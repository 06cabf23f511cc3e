// tests/gpu_probe/rt_probe.cu — TEST INFRASTRUCTURE ONLY.  Primitive-level probe of the device arithmetic.
//
// Thin kernels that evaluate the product's own device functions (csrc/rt_devmath.cuh, csrc/rt_device.cuh, the triangle repack of
// csrc/rt_repack.cuh) one primitive at a time over batches of inputs, so that tests/test_gpu_arith_contract.py can compare every
// output with the oracle's restatement (oracle/rt_oracle.cpp, orProbe, same function codes) bit for bit.  Nothing here restates a
// formula of the path: every value comes from an rtd:: function, compiled with the product's NVCC_FLAGS (tests/gpu_probe/build.py).
// The same file also compiles with g++ against the SIMT interpreter of tests/simt (-DRT_SIMT_EMU), which runs the tests on the CPU.
// The product never builds or loads this library (tests/test_host.py).
//
// Records: a case is `nin` 32-bit words in, `nout` words out (float bit patterns, or integers where the primitive takes or returns
// one).  Index mode (in == NULL): word 0 of case i is base + i * stride (mod 2^32), the other words are `partner` — the exhaustive
// scans of the scalar contract need no input arrays.  Digest: per output word, the sum over cases i < 2^32 of mix(i, word) mod 2^64, a
// NaN of a word flagged in floatMask counted as the canonical quiet NaN (NaN sign and payload are not part of the contract).
#include "../../ray_tracing_b200/csrc/rt_repack.cuh"

#include <stdio.h>
#include <vector>

namespace {

using namespace rtd;

enum ProbeFn
{
    P_LOG = 0, P_EXP = 1, P_SIN = 2, P_COS = 3, P_SINCOS = 4, P_POW = 5, P_SATURATE = 6, P_FMIN = 7, P_FMAX = 8, P_F2UINT_RZ = 9,
    P_DISPLAY_ENCODE = 10, P_NEXT_RANDOM = 11, P_RANDOM_VALUE = 12, P_RANDOM_NORMAL = 13, P_RANDOM_DIRECTION = 14,
    P_RANDOM_POINT_IN_CIRCLE = 15,
    P_RAY_BOX = 20, P_RAY_TRIANGLE = 21, P_RAY_SPHERE = 22, P_REFLECTANCE = 23, P_REFRACT = 24, P_REFLECT = 25,
    P_MATERIAL_COLOUR = 26, P_ENVIRONMENT_LIGHT = 27,
    P_MODEL_HIT = 28,                                               // device only: the model-skipping test has no counterpart in the reference
};
constexpr int P_MAX_IN = 49, P_MAX_OUT = 5;

// words in / out per case; 0 = unknown function
int arity(int fn, int& nin, int& nout)
{
    switch (fn)
    {
    case P_LOG: case P_EXP: case P_SIN: case P_COS: case P_SATURATE: case P_F2UINT_RZ: case P_DISPLAY_ENCODE: nin = 1; nout = 1; return 1;
    case P_SINCOS: case P_NEXT_RANDOM: case P_RANDOM_VALUE: case P_RANDOM_NORMAL: nin = 1; nout = 2; return 1;
    case P_POW: case P_FMIN: case P_FMAX: nin = 2; nout = 1; return 1;
    case P_RANDOM_DIRECTION: nin = 1; nout = 4; return 1;
    case P_RANDOM_POINT_IN_CIRCLE: nin = 1; nout = 3; return 1;
    case P_RAY_BOX: nin = 12; nout = 1; return 1;                  // pos, dir, boxMin, boxMax -> dst
    case P_RAY_TRIANGLE: nin = 25; nout = 5; return 1;             // pos, dir, RtTriangle (A B C nA nB nC), cull -> flags, dst, normal
    case P_RAY_SPHERE: nin = 10; nout = 2; return 1;               // pos, dir, centre, radius -> flags, dst (+inf on a miss)
    case P_REFLECTANCE: nin = 8; nout = 1; return 1;               // inDir, normal, iorA, iorB
    case P_REFRACT: nin = 8; nout = 3; return 1;
    case P_REFLECT: nin = 6; nout = 3; return 1;
    case P_MATERIAL_COLOUR: nin = 17; nout = 3; return 1;          // pos, normal, isSpecularBounce, flag, diffuse, emission, specular
    case P_ENVIRONMENT_LIGHT: nin = 11; nout = 3; return 1;        // dir, SunFocus, SunIntensity, dirToSun, SunColour
    // world pos, dir, RtTriangle, worldToLocal rows 0..2 (DevModel::w2l), geometry box lo / hi, padded world box min / max, cull
    //   -> flags (1 hit, 2 the local ray reaches the geometry box, 4 WorldBoxOutOfReach skips at bestDst = nextafter(dst, +inf)), dst
    case P_MODEL_HIT: nin = 49; nout = 2; return 1;
    default: return 0;
    }
}

__host__ __device__ inline unsigned long long mix64(unsigned long long z)        // splitmix64 finaliser
{
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
__host__ __device__ inline unsigned long long digest_term(unsigned long long i, uint32_t w, bool isFloat)
{
    if (isFloat && (w & 0x7fffffffu) > 0x7f800000u) w = 0x7fc00000u;
    return mix64((i << 32) ^ w);                              // i < 2^32 within one call: injective in (i, w)
}

RT_DI float F(uint32_t w) { return __uint_as_float(w); }
RT_DI uint32_t U(float f) { return __float_as_uint(f); }
RT_DI f3 F3(const uint32_t* a) { return make_f3(F(a[0]), F(a[1]), F(a[2])); }
RT_DI void put3(uint32_t* r, f3 v) { r[0] = U(v.x); r[1] = U(v.y); r[2] = U(v.z); }

// one case: a = the nin input words, r = the nout output words; geom / nrm / r2: the repacked triangle and r*r of the sphere
RT_DI void eval(int fn, const uint32_t* a, uint32_t* r, const TriGeom* geom, const TriNormals* nrm, float r2)
{
    switch (fn)
    {
    case P_LOG: r[0] = U(log_rt(F(a[0]))); break;
    case P_EXP: r[0] = U(exp_rt(F(a[0]))); break;
    case P_SIN: r[0] = U(sin_rt(F(a[0]))); break;
    case P_COS: r[0] = U(cos_rt(F(a[0]))); break;
    case P_SINCOS: { float s, c; sincos_rt(F(a[0]), s, c); r[0] = U(s); r[1] = U(c); break; }
    case P_POW: r[0] = U(pow_rt(F(a[0]), F(a[1]))); break;
    case P_SATURATE: r[0] = U(saturate1(F(a[0]))); break;
    case P_FMIN: r[0] = U(fminf(F(a[0]), F(a[1]))); break;
    case P_FMAX: r[0] = U(fmaxf(F(a[0]), F(a[1]))); break;
    case P_F2UINT_RZ: r[0] = __float2uint_rz(F(a[0])); break;
    case P_DISPLAY_ENCODE: r[0] = DisplayEncode(F(a[0])); break;
    case P_NEXT_RANDOM: { uint32_t s = a[0]; r[0] = NextRandom(s); r[1] = s; break; }
    case P_RANDOM_VALUE: { uint32_t s = a[0]; r[0] = U(RandomValue(s)); r[1] = s; break; }
    case P_RANDOM_NORMAL: { uint32_t s = a[0]; r[0] = U(RandomValueNormalDistribution(s)); r[1] = s; break; }
    case P_RANDOM_DIRECTION: { uint32_t s = a[0]; put3(r, RandomDirection(s)); r[3] = s; break; }
    case P_RANDOM_POINT_IN_CIRCLE: { uint32_t s = a[0]; const f2 p = RandomPointInCircle(s); r[0] = U(p.x); r[1] = U(p.y); r[2] = s; break; }
    case P_RAY_BOX:
        r[0] = U(RayBoundingBoxDst(F3(a), rcp3(F3(a + 3)), F3(a + 6), F3(a + 9)));
        break;
    case P_RAY_TRIANGLE:
    {
        // as the kernels use it: RayTriangleCore on the TriGeom record, TriangleSmoothNormal, isBackface = det < 0
        const TriGeom g = *geom;
        const TriNormals q = *nrm;
        float dst, u, v, det;
        const bool hit = RayTriangleCore(F3(a), F3(a + 3), make_f3(g.ax, g.ay, g.az), make_f3(g.abx, g.aby, g.abz), make_f3(g.acx, g.acy, g.acz),
                                         make_f3(g.nx, g.ny, g.nz), a[24] != 0u, dst, u, v, det);
        const f3 n = TriangleSmoothNormal(make_f3(q.nax, q.nay, q.naz), make_f3(q.nbx, q.nby, q.nbz), make_f3(q.ncx, q.ncy, q.ncz), u, v, det);
        r[0] = (hit ? 1u : 0u) | (det < 0.0f ? 2u : 0u);
        r[1] = U(dst);
        put3(r + 2, n);
        break;
    }
    case P_RAY_SPHERE:
    {
        float dst = 0.0f; bool inside = false;
        const bool hit = RaySphereCore(F3(a), F3(a + 3), F3(a + 6), r2, dst, inside);
        r[0] = hit ? (1u | (inside ? 2u : 0u)) : 0u;
        r[1] = hit ? U(dst) : U(inf32());
        break;
    }
    case P_REFLECTANCE: r[0] = U(CalculateReflectance(F3(a), F3(a + 3), F(a[6]), F(a[7]))); break;
    case P_REFRACT: put3(r, Refract(F3(a), F3(a + 3), F(a[6]), F(a[7]))); break;
    case P_REFLECT: put3(r, Reflect(F3(a), F3(a + 3))); break;
    case P_MATERIAL_COLOUR:
    {
        RtMaterial m;
        memset(&m, 0, sizeof(m));
        m.flag = (int)a[7];
        for (int k = 0; k < 3; k++) { m.diffuseCol[k] = F(a[8 + k]); m.emissionCol[k] = F(a[11 + k]); m.specularCol[k] = F(a[14 + k]); }
        put3(r, GetMaterialColour(&m, F3(a), F3(a + 3), a[6] != 0u));
        break;
    }
    case P_ENVIRONMENT_LIGHT:
    {
        DevParams P;
        memset(&P, 0, sizeof(P));
        P.UseSky = 1; P.SunFocus = F(a[3]); P.SunIntensity = F(a[4]);
        for (int k = 0; k < 3; k++) { P.dirToSun[k] = F(a[5 + k]); P.SunColour[k] = F(a[8 + k]); }
        put3(r, GetEnvironmentLight(P, F3(a)));
        break;
    }
    case P_MODEL_HIT:
    {
        // as the kernels run a model: ray into model space with mul_rm, RayTriangleCore on the repacked triangle, the reference's slab
        // test of the geometry box, and the world-box skip test the kernels apply before all of that
        const TriGeom g = *geom;
        float w2l[12];
        for (int k = 0; k < 12; k++) w2l[k] = F(a[24 + k]);
        const f3 pos = F3(a), dir = F3(a + 3);
        const f3 lp = mul_rm(w2l, pos, 1.0f), ld = mul_rm(w2l, dir, 0.0f);
        float dst, u, v, det;
        const bool hit = RayTriangleCore(lp, ld, make_f3(g.ax, g.ay, g.az), make_f3(g.abx, g.aby, g.abz), make_f3(g.acx, g.acy, g.acz),
                                         make_f3(g.nx, g.ny, g.nz), a[48] != 0u, dst, u, v, det);
        const bool slab = RayBoundingBoxDst(lp, rcp3(ld), F3(a + 36), F3(a + 39)) < inf32();
        const bool skip = WorldBoxOutOfReach(F3(a + 42), F3(a + 45), pos, rcp3(dir), nextafterf(dst, inf32()));
        r[0] = (hit ? 1u : 0u) | (slab ? 2u : 0u) | (skip ? 4u : 0u);
        r[1] = U(dst);
        break;
    }
    default: break;
    }
}

__global__ void k_probe(int fn, int nin, int nout, const uint32_t* __restrict__ in, uint32_t base, uint32_t stride, uint32_t partner,
                        const TriGeom* __restrict__ geom, const TriNormals* __restrict__ nrm, const float* __restrict__ r2,
                        uint32_t* __restrict__ out, uint32_t floatMask, size_t n, size_t idx0, unsigned long long* __restrict__ digest)
{
    unsigned long long h[P_MAX_OUT] = {0, 0, 0, 0, 0};
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    {
        uint32_t a[P_MAX_IN], r[P_MAX_OUT] = {0, 0, 0, 0, 0};
        if (in) { for (int k = 0; k < nin; k++) a[k] = in[i * nin + k]; }
        else { a[0] = base + (uint32_t)i * stride; for (int k = 1; k < nin; k++) a[k] = partner; }
        eval(fn, a, r, geom ? geom + i : nullptr, nrm ? nrm + i : nullptr, r2 ? r2[i] : 0.0f);
        for (int j = 0; j < nout; j++)
        {
            if (out) out[i * nout + j] = r[j];
            h[j] += digest_term(idx0 + i, r[j], (floatMask >> j) & 1u);
        }
    }
    if (digest) for (int j = 0; j < nout; j++) atomicAdd(digest + j, h[j]);
}

// One ray per thread against the TLAS in P (planned over `boxes`): TlasCollect as the kernels call it (rayInv = rcp3(dir)), then
// WorldBoxOutOfReach on every model's own box at the same bestDst.  out[3i .. 3i + 2]: the models their own box keeps, how many of
// those the TLAS mask lacks, the first of them (-1 when none).
__global__ void k_tlas_check(DevParams P, const float* __restrict__ boxes, const float* __restrict__ rays, size_t n, int* __restrict__ out)
{
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    {
        const float* r = rays + 7 * i;
        const f3 pos = make_f3(r[0], r[1], r[2]), inv = rcp3(make_f3(r[3], r[4], r[5]));
        unsigned int mask[RT_TLAS_WORDS];
        TlasCollect(P, pos, inv, r[6], mask);
        int kept = 0, lost = 0, first = -1;
        for (int m = 0; m < P.modelCount; m++)
        {
            const float* b = boxes + 6 * m;
            if (WorldBoxOutOfReach(make_f3(b[0], b[1], b[2]), make_f3(b[3], b[4], b[5]), pos, inv, r[6])) continue;
            kept++;
            if (!((mask[m >> 5] >> (m & 31)) & 1u)) { lost++; if (first < 0) first = m; }
        }
        out[3 * i] = kept; out[3 * i + 1] = lost; out[3 * i + 2] = first;
    }
}

template <class T> struct DevBuf
{
    T* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, (n ? n : 1) * sizeof(T)); }
};

int report(cudaError_t e, const char* what)
{
    if (e == cudaSuccess) return 0;
    fprintf(stderr, "rt_probe: %s: %s\n", what, cudaGetErrorString(e));
    return 2;
}

} // namespace

extern "C" {

// Evaluates `n` cases of primitive `fn` on the device.  in: n * nin words or NULL (index mode); out: n * nout words or NULL;
// digest: nout sums (see the header) or NULL.  The batch runs in slices of at most 32 MB of records, so device memory stays small.
// Returns 0, 1 for an unknown function or a wrong arity, 2 for a CUDA error (printed).
int rtpRun(int fn, int nin, int nout, const uint32_t* in, uint32_t base, uint32_t stride, uint32_t partner,
           uint32_t* out, uint32_t floatMask, size_t n, unsigned long long* digest)
{
    int ein = 0, eout = 0;
    if (!arity(fn, ein, eout) || ein != nin || eout != nout) return 1;
    if ((fn == P_RAY_TRIANGLE || fn == P_MODEL_HIT) && !in) return 1;
    const size_t slice = std::max<size_t>(1, ((size_t)32 << 20) / (4 * (size_t)(nin + nout)));
    DevBuf<uint32_t> dIn, dOut; DevBuf<unsigned long long> dDig; DevBuf<RtTriangle> dTri; DevBuf<TriGeom> dGeom; DevBuf<TriNormals> dNrm; DevBuf<float> dR2;
    const size_t m0 = std::min(n, slice);
    if (in && report(dIn.alloc(m0 * nin), "cudaMalloc")) return 2;
    if (out && report(dOut.alloc(m0 * nout), "cudaMalloc")) return 2;
    if (report(dDig.alloc(P_MAX_OUT), "cudaMalloc")) return 2;
    if ((fn == P_RAY_TRIANGLE || fn == P_MODEL_HIT) && (report(dTri.alloc(m0), "cudaMalloc") || report(dGeom.alloc(m0), "cudaMalloc") || report(dNrm.alloc(m0), "cudaMalloc"))) return 2;
    if (fn == P_RAY_SPHERE && report(dR2.alloc(m0), "cudaMalloc")) return 2;
    if (report(cudaMemset(dDig.p, 0, P_MAX_OUT * sizeof(unsigned long long)), "cudaMemset")) return 2;
    std::vector<RtTriangle> tris; std::vector<float> r2;
    for (size_t s = 0; s < n; s += slice)
    {
        const size_t m = std::min(slice, n - s);
        if (in && report(cudaMemcpy(dIn.p, in + s * nin, m * nin * 4, cudaMemcpyHostToDevice), "cudaMemcpy")) return 2;
        if (fn == P_RAY_TRIANGLE || fn == P_MODEL_HIT)
        {
            // the reference-layout triangles go through the product's upload repack, as rtSetBuffer("Triangles") does
            tris.resize(m);
            for (size_t i = 0; i < m; i++) memcpy(&tris[i], in + (s + i) * nin + 6, sizeof(RtTriangle));
            if (report(cudaMemcpy(dTri.p, tris.data(), m * sizeof(RtTriangle), cudaMemcpyHostToDevice), "cudaMemcpy")) return 2;
            RT_LAUNCH((unsigned)((m + 255) / 256), 256, 0, (cudaStream_t)0, k_repack_tris, dTri.p, dGeom.p, dNrm.p, m);
        }
        if (fn == P_RAY_SPHERE)
        {
            // r*r as buildSpheres forms it (rt_repack.cuh sphereR2)
            r2.resize(m);
            for (size_t i = 0; i < m; i++) { float rad; memcpy(&rad, in + (s + i) * nin + 9, 4); r2[i] = sphereR2(rad); }
            if (report(cudaMemcpy(dR2.p, r2.data(), m * 4, cudaMemcpyHostToDevice), "cudaMemcpy")) return 2;
        }
#ifdef RT_SIMT_EMU
        const unsigned grid = (unsigned)std::min<size_t>((m + 255) / 256, 16);     // few fibers, each looping: the interpreter's cost is per thread
#else
        const unsigned grid = (unsigned)std::min<size_t>((m + 255) / 256, 8192);
#endif
        RT_LAUNCH(grid, 256, 0, (cudaStream_t)0, k_probe, fn, nin, nout, in ? dIn.p : nullptr, base + (uint32_t)s * stride, stride, partner,
                  dGeom.p, dNrm.p, dR2.p, out ? dOut.p : nullptr, floatMask, m, s, digest ? dDig.p : nullptr);
        if (report(cudaGetLastError(), "launch")) return 2;
        if (out && report(cudaMemcpy(out + s * nout, dOut.p, m * nout * 4, cudaMemcpyDeviceToHost), "cudaMemcpy")) return 2;
    }
    if (digest)
    {
        unsigned long long part[P_MAX_OUT];
        if (report(cudaMemcpy(part, dDig.p, sizeof(part), cudaMemcpyDeviceToHost), "cudaMemcpy")) return 2;
        for (int j = 0; j < nout; j++) digest[j] += part[j];
    }
    return report(cudaStreamSynchronize((cudaStream_t)0), "cudaStreamSynchronize");
}

// The product's padded boxes (host code of rt_repack.cuh, no device work).  Sphere i: centreRadius[4i..4i+3] -> lo / hi[3i..3i+2], the
// box buildSpheres gives it for ray origins in the box origin[6i..6i+2] .. origin[6i+3..6i+5].
void rtpSphereBoxes(const float* centreRadius, const float* origin, float* lo, float* hi, size_t n)
{
    for (size_t i = 0; i < n; i++) paddedSphereBox(centreRadius + 4 * i, centreRadius[4 * i + 3], origin + 6 * i, origin + 6 * i + 3, lo + 3 * i, hi + 3 * i);
}
// Model i: worldToLocal (column-major, 16 floats) and the mesh's geometry box geo[6i..6i+5] (lo, hi) -> the exact world box of that
// geometry (double, exact[6i..]) and the padded world box buildModels stores in DevModel (padded[6i..]) for ray origins in the box
// origin[6i..6i+5]; returns the number of models placed.
int rtpModelBoxes(const float* worldToLocal, const float* geo, const float* origin, double* exact, float* padded, size_t n)
{
    int placedCount = 0;
    for (size_t i = 0; i < n; i++)
    {
        const double originPad = originPadOf(origin + 6 * i, origin + 6 * i + 3);
        RtModel m;
        memset(&m, 0, sizeof(m));
        memcpy(m.worldToLocal, worldToLocal + 16 * i, 64);
        MeshRoot root{};
        for (int a = 0; a < 3; a++) { root.geoLo[a] = geo[6 * i + a]; root.geoHi[a] = geo[6 * i + 3 + a]; }
        root.geoValid = true;
        const bool placed = RepackState::worldBoxOfModel(m, root, exact + 6 * i, exact + 6 * i + 3);
        paddedModelBox(placed, exact + 6 * i, exact + 6 * i + 3, originPad, padded + 6 * i, padded + 6 * i + 3);
        placedCount += placed ? 1 : 0;
    }
    return placedCount;
}

// The TLAS over n model world boxes (boxes[6m..6m+5]: min xyz, max xyz, as DevModel holds them), planned by the host's
// RepackState::planTlas (the tree rtxPlanTlas exposes), walked on the device by TlasCollect for each of the nrays rays (rays[7i..]:
// pos, dir, bestDst); see k_tlas_check for out.  Returns 0, 1 for n outside 1 .. RT_TLAS_MAX_MODELS, 2 for a CUDA error (printed).
int rtpTlasCheck(const float* boxes, int n, const float* rays, size_t nrays, int* out)
{
    if (n < 1 || n > RT_TLAS_MAX_MODELS) return 1;
    std::vector<DevModel> dm((size_t)n);
    for (int i = 0; i < n; i++)
    {
        memset(&dm[i], 0, sizeof(DevModel));
        const float* b = boxes + 6 * i;
        dm[i].wmin[0] = b[0]; dm[i].wmin[1] = b[1]; dm[i].wmin[2] = b[2]; dm[i].wmaxx = b[3]; dm[i].wmaxy = b[4]; dm[i].wmaxz = b[5];
    }
    std::vector<NodePair> pairs; std::vector<int> order;
    DevParams P;
    memset(&P, 0, sizeof(P));
    P.modelCount = n;
    RepackState::planTlas(dm, n, pairs, order, P.tlasRootStart, P.tlasRootCount);
    DevBuf<NodePair> dPairs; DevBuf<int> dLeaves, dOut; DevBuf<float> dBoxes, dRays;
    if (report(dPairs.alloc(pairs.size()), "cudaMalloc") || report(dLeaves.alloc(order.size()), "cudaMalloc") || report(dOut.alloc(3 * nrays), "cudaMalloc") ||
        report(dBoxes.alloc(6 * (size_t)n), "cudaMalloc") || report(dRays.alloc(7 * nrays), "cudaMalloc")) return 2;
    if ((!pairs.empty() && report(cudaMemcpy(dPairs.p, pairs.data(), pairs.size() * sizeof(NodePair), cudaMemcpyHostToDevice), "cudaMemcpy")) ||
        report(cudaMemcpy(dLeaves.p, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice), "cudaMemcpy") ||
        report(cudaMemcpy(dBoxes.p, boxes, 6 * (size_t)n * 4, cudaMemcpyHostToDevice), "cudaMemcpy") ||
        (nrays && report(cudaMemcpy(dRays.p, rays, 7 * nrays * 4, cudaMemcpyHostToDevice), "cudaMemcpy"))) return 2;
    P.tlasPairs = dPairs.p; P.tlasLeaves = dLeaves.p; P.tlas = 1;
    if (!nrays) return 0;
#ifdef RT_SIMT_EMU
    const unsigned grid = (unsigned)std::min<size_t>((nrays + 255) / 256, 16);
#else
    const unsigned grid = (unsigned)std::min<size_t>((nrays + 255) / 256, 8192);
#endif
    RT_LAUNCH(grid, 256, 0, (cudaStream_t)0, k_tlas_check, P, dBoxes.p, dRays.p, nrays, dOut.p);
    if (report(cudaGetLastError(), "launch")) return 2;
    if (report(cudaMemcpy(out, dOut.p, 3 * nrays * 4, cudaMemcpyDeviceToHost), "cudaMemcpy")) return 2;
    return report(cudaStreamSynchronize((cudaStream_t)0), "cudaStreamSynchronize");
}

} // extern "C"
