// rt_repack.cuh — upload-time repack of the reference-layout buffers into the streams the wavefront
// kernel reads (records defined in rt_device.cuh), plus the multi-GPU tile pack / unpack kernels.
//
//  Nodes (32 B, depth-first order of the reference builder, BVH.cs:89-181)
//      -> NodePair (64 B, 64-B aligned): the two children of one inner node, numbered breadth-first per
//         mesh; the first `hot` pairs of every mesh are gathered at the front of the array so the top of
//         every tree is ONE contiguous range that a single TMA bulk copy stages into shared memory.
//         Child order (A = first child, B = second) and therefore the traversal order are unchanged.
//  Triangles (72 B) -> TriGeom (48 B: A, AB, AC, cross(AB,AC)) + TriNormals (48 B), same triangle order.
//  ModelInfo (224 B) -> DevModel (128 B): matrix rows, BVH root, cull flag, material index.
//  Spheres (104 B)   -> DevSphere (32 B): centre, radius, r*r.
#pragma once
#include "rt_device.cuh"
#include <algorithm>
#include <cmath>
#include <map>
#include <string>
#include <utility>
#include <vector>

namespace rtd {

__global__ void k_repack_tris(const RtTriangle* __restrict__ in, TriGeom* __restrict__ geom, TriNormals* __restrict__ nrm, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const RtTriangle t = in[i];
    const f3 A = load3(t.posA), B = load3(t.posB), C = load3(t.posC);
    const f3 edgeAB = B - A, edgeAC = C - A;            // HL:190-191
    const f3 N = cross3(edgeAB, edgeAC);                // HL:192
    TriGeom g;
    g.ax = A.x; g.ay = A.y; g.az = A.z; g.abx = edgeAB.x; g.aby = edgeAB.y; g.abz = edgeAB.z;
    g.acx = edgeAC.x; g.acy = edgeAC.y; g.acz = edgeAC.z; g.nx = N.x; g.ny = N.y; g.nz = N.z;
#ifdef RT_TRI_PAD64
    g.pad[0] = g.pad[1] = g.pad[2] = g.pad[3] = 0.0f;
#endif
    geom[i] = g;
    TriNormals q;
    q.nax = t.normA[0]; q.nay = t.normA[1]; q.naz = t.normA[2];
    q.nbx = t.normB[0]; q.nby = t.normB[1]; q.nbz = t.normB[2];
    q.ncx = t.normC[0]; q.ncy = t.normC[1]; q.ncz = t.normC[2];
    q.pad0 = q.pad1 = q.pad2 = 0.0f;
    nrm[i] = q;
}

template <class T> struct RBuf
{
    T* p = nullptr; size_t cap = 0;
    cudaError_t ensure(size_t n) { if (n <= cap && p) return cudaSuccess; if (p) cudaFree(p); p = nullptr; cap = 0; if (!n) return cudaSuccess; cudaError_t e = cudaMalloc(&p, n * sizeof(T)); if (e == cudaSuccess) cap = n; return e; }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// geo: the box a ray must touch to hit anything of the mesh, in mesh space — the union of the root's two child boxes (the reference
// tests only child boxes, HL:257-270, never the root's own bounds) or, for a root that is a leaf, the bounds of its triangles'
// vertices; geoValid = false when any of those numbers is not finite (such a model is never skipped).
// Host staging that outlives the call that fills it: pinned memory + an event recorded behind the copies that read it, so that a
// per-frame rebuild (the reference re-sends ModelInfo every frame, RCM:192-204) waits for its own previous COPY only — never for
// the trace kernel queued behind it, which a cudaStreamSynchronize on a local vector did.
template <class T> struct PinnedStage
{
    T* p = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool pending = false;
    cudaError_t acquire(size_t n)
    {
        cudaError_t e;
        if (pending) { if ((e = cudaEventSynchronize(ev)) != cudaSuccess) return e; pending = false; }
        if (n <= cap && p) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        if ((e = cudaMallocHost((void**)&p, std::max<size_t>(n, 1) * sizeof(T))) != cudaSuccess) return e;
        cap = std::max<size_t>(n, 1);
        return cudaSuccess;
    }
    cudaError_t commit(cudaStream_t stream)
    {
        cudaError_t e;
        if (!ev && (e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming)) != cudaSuccess) return e;
        if ((e = cudaEventRecord(ev, stream)) != cudaSuccess) return e;
        pending = true; return cudaSuccess;
    }
    void release() { if (pending && ev) cudaEventSynchronize(ev); pending = false; if (p) cudaFreeHost(p); p = nullptr; cap = 0; if (ev) cudaEventDestroy(ev); ev = nullptr; }
};

struct MeshRoot { int rootStart, rootCount; float geoLo[3], geoHi[3]; bool geoValid; int leafRootTriStart; };

// Host only: binary tree over n axis-aligned boxes in NodePair records (two child boxes per record; count > 0 <=> leaf whose
// items are order[start .. start + count)).  Median split of the item centres on the widest centre axis (ties by item index, so
// the tree is a function of the input alone), leaves of at most `leafSize` items, records emitted parent before children —
// depth <= ceil(log2(n / leafSize)) + 1.  Used for the sphere accelerator and for the TLAS over the models' world boxes; both
// only decide what a ray may skip, so its shape never changes a result.
//
// sahDepth > 0 (the TLAS): down to that depth a range is split where the surface-area heuristic is smallest — all three axes, every
// position of the items sorted by centre, cost = area(left) x count + area(right) x count — which keeps the boxes of a level apart
// much better than the median does when the items are scattered; below it the median split bounds the depth (<= sahDepth +
// log2(n / leafSize) + 1, the device walk keeps a stack of RT_TLAS_STACK entries and marks everything if that ever overflowed).
inline void BuildMedianSplitPairs(const std::vector<float>& lo, const std::vector<float>& hi, const std::vector<float>& cen, size_t n, int leafSize,
                                  std::vector<int>& order, std::vector<NodePair>& pairsOut, int& rootStart, int& rootCount, int sahDepth = 0)
{
    order.resize(n);
    for (size_t i = 0; i < n; i++) order[i] = (int)i;
    pairsOut.clear(); pairsOut.reserve(n);
    auto boundsOf = [&](int start, int count, float blo[3], float bhi[3]) {
        for (int a = 0; a < 3; a++) { blo[a] = INFINITY; bhi[a] = -INFINITY; }
        for (int k = start; k < start + count; k++) for (int a = 0; a < 3; a++) { blo[a] = std::min(blo[a], lo[3 * order[k] + a]); bhi[a] = std::max(bhi[a], hi[3 * order[k] + a]); }
    };
    struct Work { int pairIndex, side, start, count, depth; };
    std::vector<Work> work;
    auto halfArea = [](const float blo[3], const float bhi[3]) -> double {
        const double x = (double)bhi[0] - blo[0], y = (double)bhi[1] - blo[1], z = (double)bhi[2] - blo[2];
        const double a = x * y + x * z + y * z;
        return a == a ? a : INFINITY;                                      // infinite boxes (inf - inf, inf x 0): as bad as it gets
    };
    std::vector<double> suffixArea;
    auto splitRangeSah = [&](int start, int count) -> int {
        // returns the first index of the right part after sorting the range along the best axis, or -1 if no split separates anything
        double best = INFINITY; int bestAxis = -1, bestK = -1;
        suffixArea.resize((size_t)count + 1);
        for (int axis = 0; axis < 3; axis++)
        {
            std::sort(order.begin() + start, order.begin() + start + count,
                      [&](int x, int y) { return cen[3 * x + axis] < cen[3 * y + axis] || (cen[3 * x + axis] == cen[3 * y + axis] && x < y); });
            float blo[3] = {INFINITY, INFINITY, INFINITY}, bhi[3] = {-INFINITY, -INFINITY, -INFINITY};
            for (int k = count - 1; k >= 1; k--)
            {
                for (int a = 0; a < 3; a++) { blo[a] = std::min(blo[a], lo[3 * order[start + k] + a]); bhi[a] = std::max(bhi[a], hi[3 * order[start + k] + a]); }
                suffixArea[k] = halfArea(blo, bhi);
            }
            for (int a = 0; a < 3; a++) { blo[a] = INFINITY; bhi[a] = -INFINITY; }
            for (int k = 1; k < count; k++)                               // left = first k items of the sorted range
            {
                for (int a = 0; a < 3; a++) { blo[a] = std::min(blo[a], lo[3 * order[start + k - 1] + a]); bhi[a] = std::max(bhi[a], hi[3 * order[start + k - 1] + a]); }
                const double cost = halfArea(blo, bhi) * k + suffixArea[k] * (count - k);
                if (cost < best) { best = cost; bestAxis = axis; bestK = k; }
            }
        }
        if (bestAxis < 0) return -1;
        if (bestAxis != 2)
            std::sort(order.begin() + start, order.begin() + start + count,
                      [&](int x, int y) { return cen[3 * x + bestAxis] < cen[3 * y + bestAxis] || (cen[3 * x + bestAxis] == cen[3 * y + bestAxis] && x < y); });
        return start + bestK;
    };
    auto splitRange = [&](int start, int count) -> int {
        float clo[3] = {INFINITY, INFINITY, INFINITY}, chi[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int k = start; k < start + count; k++) for (int a = 0; a < 3; a++) { clo[a] = std::min(clo[a], cen[3 * order[k] + a]); chi[a] = std::max(chi[a], cen[3 * order[k] + a]); }
        int axis = 0; for (int a = 1; a < 3; a++) if (chi[a] - clo[a] > chi[axis] - clo[axis]) axis = a;
        const int mid = start + count / 2;
        std::nth_element(order.begin() + start, order.begin() + mid, order.begin() + start + count,
                         [&](int x, int y) { return cen[3 * x + axis] < cen[3 * y + axis] || (cen[3 * x + axis] == cen[3 * y + axis] && x < y); });
        return mid;
    };
    if ((int)n <= leafSize) { rootStart = 0; rootCount = (int)n; return; }
    rootStart = 0; rootCount = 0;
    pairsOut.push_back(NodePair());
    work.push_back(Work{0, -1, 0, (int)n, 0});
    for (size_t w = 0; w < work.size(); w++)
    {
        const Work cur = work[w];
        int mid = cur.depth < sahDepth ? splitRangeSah(cur.start, cur.count) : -1;
        if (mid < 0) mid = splitRange(cur.start, cur.count);
        const int cs[2] = {cur.start, mid}, cc[2] = {mid - cur.start, cur.start + cur.count - mid};
        for (int side = 0; side < 2; side++)
        {
            float blo[3], bhi[3];
            boundsOf(cs[side], cc[side], blo, bhi);
            int st, ct;
            if (cc[side] <= leafSize) { st = cs[side]; ct = cc[side]; }
            else { st = (int)pairsOut.size(); ct = 0; pairsOut.push_back(NodePair()); work.push_back(Work{st, side, cs[side], cc[side], cur.depth + 1}); }
            NodePair& q = pairsOut[cur.pairIndex];       // (push_back may have moved the vector)
            if (side == 0) { q.aMinX = blo[0]; q.aMinY = blo[1]; q.aMinZ = blo[2]; q.aMaxX = bhi[0]; q.aMaxY = bhi[1]; q.aMaxZ = bhi[2]; q.aStart = st; q.aCount = ct; }
            else           { q.bMinX = blo[0]; q.bMinY = blo[1]; q.bMinZ = blo[2]; q.bMaxX = bhi[0]; q.bMaxY = bhi[1]; q.bMaxZ = bhi[2]; q.bStart = st; q.bCount = ct; }
        }
    }
}

// The most entries a stack walk of a BuildMedianSplitPairs tree over n items can hold (one per inner node above a leaf, rounded up):
// sahDepth + ceil(log2 n) + 1.
constexpr int SplitTreeStackBound(long long n, int sahDepth)
{
    int lg = 0;
    while (lg < 62 && (1LL << lg) < n) lg++;
    return sahDepth + lg + 1;
}

#ifndef RT_ORIGIN_PAD_SCALE
#define RT_ORIGIN_PAD_SCALE 2e-5      // of the largest coordinate R a ray origin can have (~170 ulp(R)); see buildModels.  Measured on the interpreter
                                      // build: 144 differing values with 0, none with 1e-7 (about 1 ulp) and above; the error estimate is <= 40 ulp(R)
#endif

// Padding of a model's world box (RepackState::buildModels; the reasoning is there).  originPadOf: the part that covers rays starting far
// away, RT_ORIGIN_PAD_SCALE of the largest coordinate of the origin box (infinite when that box is not finite).  paddedModelBox: the
// box handed to WorldBoxOutOfReach for the exact world box lo..hi of the model's geometry (placed = false: nothing is known, +-inf).
inline double originPadOf(const float originLo[3], const float originHi[3])
{
    double originExtent = 0;
    for (int a = 0; a < 3; a++)
    {
        originExtent = std::max(originExtent, std::max(std::fabs((double)originLo[a]), std::fabs((double)originHi[a])));
        if (!std::isfinite(originLo[a]) || !std::isfinite(originHi[a])) originExtent = INFINITY;
    }
    return RT_ORIGIN_PAD_SCALE * originExtent;
}
inline void paddedModelBox(bool placed, const double lo[3], const double hi[3], double originPad, float bmin[3], float bmax[3])
{
    for (int a = 0; a < 3; a++)
    {
        const double pad = placed ? 1e-4 * ((hi[a] - lo[a]) + std::fabs(lo[a]) + std::fabs(hi[a])) + 1e-5 + originPad : (double)INFINITY;
        if (!std::isfinite(pad)) { bmin[a] = -INFINITY; bmax[a] = INFINITY; continue; }
        bmin[a] = std::nextafterf((float)(lo[a] - pad), -INFINITY); bmax[a] = std::nextafterf((float)(hi[a] + pad), INFINITY);
    }
}

// r*r of a sphere as DevSphere::r2 holds it: one host multiply (HL:299).  Host code is built without FMA contraction, so this is that product.
inline float sphereR2(float radius) { volatile float r = radius; return r * r; }

// Box of sphere (centre, radius) in the sphere accelerator (RepackState::buildSpheres): the reference's discriminant carries an absolute
// error of at most ~2e-6 (D^2 + r^2) (D = distance from the ray origin to the centre), which moves a computed hit point about
// 2.5e-7 (D^2 + r^2) / r off the sphere (measured worst 2.53e-7, DESIGN.md §5); pad by 16 * 2^-23 * (Dmax^2 + r^2) / r (7.5x that)
// plus 1e-5 of the scene size for the slab test itself.  originLo / originHi: a box containing every possible ray origin.
inline void paddedSphereBox(const float centre[3], float radius, const float originLo[3], const float originHi[3], float lo[3], float hi[3])
{
    double sceneSize = 0;
    for (int a = 0; a < 3; a++) sceneSize = std::max(sceneSize, (double)originHi[a] - originLo[a]);
    double dmax2 = 0;
    for (int a = 0; a < 3; a++)
    {
        const double c = centre[a];
        const double far = std::max(std::fabs(c - originLo[a]), std::fabs(c - originHi[a]));
        dmax2 += far * far;
    }
    const double r = std::fabs((double)radius);
    const double pad = 16.0 * 1.1920929e-7 * (dmax2 + r * r) / std::max(r, 1e-30) + 1e-5 * sceneSize + 1e-6;
    for (int a = 0; a < 3; a++)
    {
        lo[a] = (float)(centre[a] - r - pad); hi[a] = (float)(centre[a] + r + pad);
        lo[a] = std::nextafterf(lo[a], -INFINITY); hi[a] = std::nextafterf(hi[a], INFINITY);
    }
}

struct RepackState
{
    RBuf<NodePair> pairs; RBuf<TriGeom> triGeom; RBuf<TriNormals> triNormals; RBuf<DevModel> models; RBuf<DevSphere> spheres;
    std::map<std::pair<int,int>, MeshRoot> roots;     // (nodeOffset, triOffset) -> encoded root
    int smemPairs = 0;
    int budgetUsed = -1;
    bool flagsUsed = false;                         // references to treelet roots carry bit 30 (RT_TREELET_PREFETCH builds only)
    int orderUsed = 0;                              // treeletDepth of the current pair layout
    size_t totalPairs = 0;

    void release() { pairs.release(); triGeom.release(); triNormals.release(); models.release(); spheres.release(); sphPairs.release(); sphLeaves.release(); tlasPairs.release(); tlasLeaves.release(); tlas = 0; roots.clear(); stageModels.release(); stageSpheres.release(); stageTlasPairs.release(); stageTlasLeaves.release(); }

    // Renumbering of every distinct mesh referenced by the first modelCount models.  Host only (no CUDA call):
    // fills `out`, `roots`, `smemPairs`, `totalPairs`; a non-empty `msg` reports a malformed BVH.
    // Record order inside a mesh (it changes where records live, never what a traversal visits):
    //   treeletDepth = 0   breadth-first (the default: the top of the tree is one contiguous range)
    //   treeletDepth = d   treelets of d levels, breadth-first inside a treelet, treelets in depth-first order (first child's
    //                      subtree first): a descent stays inside one or two 128-byte lines for d levels, and with d = 1
    //                      (plain pre-order) the record of child A directly follows its parent's.  The first `hot` records
    //                      (shared-memory staging) stay the breadth-first top whatever the order of the rest.
    void planScene(const std::vector<RtNode>& nodes, const std::vector<RtModel>& mdl, int modelCount, size_t triCount, int smemOpt,
                   std::vector<NodePair>& out, std::string& msg, int treeletDepth = 0, bool flagTreeletRoots = false)
    {
        roots.clear(); smemPairs = 0; totalPairs = 0; out.clear();
        struct Mesh { int nodeOffset, triOffset; std::vector<int> order; /* global node index of first child, in BFS pair order */
                      std::vector<int> kidA, kidB; /* BFS pair id of the inner children of pair k, -1 for a leaf */
                      std::vector<int> perm; /* BFS pair id -> position inside the mesh */ std::vector<char> troot; /* first record of a treelet */ size_t hot = 0, hotBase = 0, coldBase = 0; };
        std::vector<Mesh> meshes;
        for (int i = 0; i < modelCount; i++)
        {
            const std::pair<int,int> key(mdl[i].nodeOffset, mdl[i].triOffset);
            if (roots.count(key)) continue;
            roots[key] = MeshRoot{};
            Mesh m; m.nodeOffset = key.first; m.triOffset = key.second;
            const RtNode& root = nodes[m.nodeOffset];
            if (root.triangleCount <= 0)
            {
                // BFS over inner nodes; order[k] = global index of the first child of the k-th inner node met
                std::vector<int> queue, level; queue.push_back(m.nodeOffset); level.push_back(1);
                for (size_t q = 0; q < queue.size(); q++)
                {
                    const RtNode& nd = nodes[queue[q]];
                    const long long a = (long long)m.nodeOffset + nd.startIndex;
                    if (a < 0 || a + 1 >= (long long)nodes.size()) { msg = "BVH child index out of range"; return; }
                    if (queue.size() > nodes.size()) { msg = "BVH has a cycle"; return; }
                    // every traversal stack of the kernels (and the oracle's) holds RT_MAX_BVH_DEPTH + 1 entries; the reference's builder stops at 32 (BVH.cs:91)
                    if (level[q] > RT_MAX_BVH_DEPTH) { msg = "BVH too deep: more than 63 levels of inner nodes (the traversal stacks hold 64 entries; the reference's builder stops at 32)"; return; }
                    m.order.push_back((int)a);
                    if (nodes[a].triangleCount <= 0) { m.kidA.push_back((int)queue.size()); queue.push_back((int)a); level.push_back(level[q] + 1); } else m.kidA.push_back(-1);
                    if (nodes[a + 1].triangleCount <= 0) { m.kidB.push_back((int)queue.size()); queue.push_back((int)a + 1); level.push_back(level[q] + 1); } else m.kidB.push_back(-1);
                }
            }
            meshes.push_back(std::move(m));
        }
        for (auto& m : meshes) totalPairs += m.order.size();

        // shared-memory budget (pairs) split over the meshes by water-filling, smallest mesh first
        size_t budget = smemOpt < 0 ? 0 : (size_t)smemOpt;
        if (budget > 3072) budget = 3072;                                   // 192 KB of the 227 KB a CTA may own
        budgetUsed = (int)budget;
        {
            std::vector<size_t> idx(meshes.size());
            for (size_t i = 0; i < idx.size(); i++) idx[i] = i;
            std::sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return meshes[a].order.size() < meshes[b].order.size(); });
            size_t left = budget;
            for (size_t k = 0; k < idx.size(); k++)
            {
                const size_t share = left / (idx.size() - k);
                Mesh& m = meshes[idx[k]];
                m.hot = std::min(share, m.order.size());
                left -= m.hot;
            }
        }
        size_t hotTotal = 0; for (auto& m : meshes) { m.hotBase = hotTotal; hotTotal += m.hot; }
        size_t coldTotal = hotTotal; for (auto& m : meshes) { m.coldBase = coldTotal; coldTotal += m.order.size() - m.hot; }
        smemPairs = (int)hotTotal;

        out.assign(totalPairs, NodePair());
        for (auto& m : meshes)
        {
            // position of every pair inside the mesh
            const size_t n = m.order.size();
            m.perm.assign(n, -1);
            m.troot.assign(n, 0);
            if (treeletDepth <= 0) for (size_t k = 0; k < n; k++) m.perm[k] = (int)k;
            else if (n > 0)
            {
                int next = (int)m.hot;
                for (size_t k = 0; k < m.hot; k++) m.perm[k] = (int)k;
                std::vector<int> todo(1, 0), level, below;                 // treelet roots still to lay out (depth-first: a stack)
                while (!todo.empty())
                {
                    level.assign(1, todo.back()); todo.pop_back();
                    m.troot[level[0]] = 1;
                    for (int d = 0; d < treeletDepth && !level.empty(); d++)
                    {
                        below.clear();
                        for (int k : level)
                        {
                            if (m.perm[k] < 0) m.perm[k] = next++;
                            if (m.kidA[k] >= 0) below.push_back(m.kidA[k]);
                            if (m.kidB[k] >= 0) below.push_back(m.kidB[k]);
                        }
                        level.swap(below);
                    }
                    for (size_t i = level.size(); i-- > 0;) todo.push_back(level[i]);     // leftmost treelet next
                }
            }
            // (with flagTreeletRoots a reference to the first record of a treelet carries bit 30, see LoadPair)
            auto globalPair = [&](size_t bfsId) { const size_t local = (size_t)m.perm[bfsId]; const int g = (int)(local < m.hot ? m.hotBase + local : m.coldBase + (local - m.hot));
                                                  return (flagTreeletRoots && m.troot[bfsId]) ? (g | 0x40000000) : g; };
            auto slotOf = [&](size_t bfsId) { const size_t local = (size_t)m.perm[bfsId]; return (size_t)(local < m.hot ? m.hotBase + local : m.coldBase + (local - m.hot)); };
            // second pass in BFS order: the k-th inner node met owns pair k; its inner children are the next ones the BFS met
            size_t nextChildPair = 1;       // pair 0 belongs to the root
            const RtNode& root = nodes[m.nodeOffset];
            MeshRoot r{};
            r.leafRootTriStart = -1;
            if (root.triangleCount > 0)
            {
                r.rootStart = m.triOffset + root.startIndex; r.rootCount = root.triangleCount;
                r.leafRootTriStart = r.rootStart; r.geoValid = false;               // buildScene reads the triangles back and fills the box
            }
            else
            {
                r.rootStart = globalPair(0); r.rootCount = 0;
                const RtNode& A = nodes[m.order[0]]; const RtNode& B = nodes[m.order[0] + 1];
                r.geoValid = true;
                for (int a = 0; a < 3; a++)
                {
                    r.geoLo[a] = std::min(A.boundsMin[a], B.boundsMin[a]); r.geoHi[a] = std::max(A.boundsMax[a], B.boundsMax[a]);
                    if (!std::isfinite(A.boundsMin[a]) || !std::isfinite(B.boundsMin[a]) || !std::isfinite(A.boundsMax[a]) || !std::isfinite(B.boundsMax[a])) r.geoValid = false;
                }
            }
            roots[std::make_pair(m.nodeOffset, m.triOffset)] = r;
            for (size_t k = 0; k < m.order.size(); k++)
            {
                const RtNode& A = nodes[m.order[k]];
                const RtNode& B = nodes[m.order[k] + 1];
                NodePair p;
                p.aMinX = A.boundsMin[0]; p.aMinY = A.boundsMin[1]; p.aMinZ = A.boundsMin[2];
                p.aMaxX = A.boundsMax[0]; p.aMaxY = A.boundsMax[1]; p.aMaxZ = A.boundsMax[2];
                p.bMinX = B.boundsMin[0]; p.bMinY = B.boundsMin[1]; p.bMinZ = B.boundsMin[2];
                p.bMaxX = B.boundsMax[0]; p.bMaxY = B.boundsMax[1]; p.bMaxZ = B.boundsMax[2];
                if (A.triangleCount > 0) { p.aStart = m.triOffset + A.startIndex; p.aCount = A.triangleCount; if (p.aStart < 0 || (size_t)p.aStart + p.aCount > triCount) { msg = "BVH leaf triangle range out of bounds"; return; } }
                else { p.aStart = globalPair(nextChildPair++); p.aCount = 0; }
                if (B.triangleCount > 0) { p.bStart = m.triOffset + B.startIndex; p.bCount = B.triangleCount; if (p.bStart < 0 || (size_t)p.bStart + p.bCount > triCount) { msg = "BVH leaf triangle range out of bounds"; return; } }
                else { p.bStart = globalPair(nextChildPair++); p.bCount = 0; }
                out[slotOf(k)] = p;
            }
            if (root.triangleCount > 0 && ((size_t)r.rootStart + r.rootCount > triCount)) { msg = "BVH root triangle range out of bounds"; return; }
        }
    }

    cudaError_t buildScene(const std::vector<RtNode>& nodes, const std::vector<RtModel>& mdl, int modelCount,
                           const RtTriangle* dTris, size_t triCount, int smemOpt, cudaStream_t stream, std::string& msg, int treeletDepth = 0,
                           bool flagTreeletRoots = false)
    {
        std::vector<NodePair> out;
        planScene(nodes, mdl, modelCount, triCount, smemOpt, out, msg, treeletDepth, flagTreeletRoots);
        orderUsed = treeletDepth; flagsUsed = flagTreeletRoots;
        if (!msg.empty()) return cudaSuccess;
        cudaError_t e;
        if ((e = pairs.ensure(std::max<size_t>(totalPairs, 1))) != cudaSuccess) return e;
        if (totalPairs && (e = cudaMemcpyAsync(pairs.p, out.data(), totalPairs * sizeof(NodePair), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;      // `out` is a local
        for (auto& kv : roots)                                                  // meshes whose root is a leaf: the box of its triangles' vertices
        {
            MeshRoot& r = kv.second;
            if (r.leafRootTriStart < 0 || r.rootCount <= 0) continue;
            std::vector<RtTriangle> t((size_t)r.rootCount);
            if ((e = cudaMemcpyAsync(t.data(), dTris + r.leafRootTriStart, t.size() * sizeof(RtTriangle), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
            if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
            r.geoValid = true;
            for (int a = 0; a < 3; a++) { r.geoLo[a] = INFINITY; r.geoHi[a] = -INFINITY; }
            for (const RtTriangle& q : t) for (int a = 0; a < 3; a++)
            {
                const float v[3] = {q.posA[a], q.posB[a], q.posC[a]};
                for (float x : v) { if (!std::isfinite(x)) r.geoValid = false; r.geoLo[a] = std::min(r.geoLo[a], x); r.geoHi[a] = std::max(r.geoHi[a], x); }
            }
        }
        if ((e = triGeom.ensure(std::max<size_t>(triCount, 1))) != cudaSuccess) return e;
        if ((e = triNormals.ensure(std::max<size_t>(triCount, 1))) != cudaSuccess) return e;
        if (triCount)
        {
            RT_LAUNCH((unsigned)((triCount + 255) / 256), 256, 0, stream, k_repack_tris, dTris, triGeom.p, triNormals.p, triCount);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
        }
        return cudaSuccess;
    }

    // ---- TLAS over the models' padded world boxes (SURVEY 8f #3) --------------------------------------------------------------
    // Rebuilt with the model records, i.e. whenever ModelInfo is re-sent (the reference re-sends it every frame, RCM:192-204): a
    // median-split tree over a few hundred to a few thousand boxes is microseconds of host work next to a frame.
    RBuf<NodePair> tlasPairs; RBuf<int> tlasLeaves;
    PinnedStage<DevModel> stageModels; PinnedStage<DevSphere> stageSpheres; PinnedStage<NodePair> stageTlasPairs; PinnedStage<int> stageTlasLeaves;
    int tlas = 0, tlasRootStart = 0, tlasRootCount = 0;
#ifndef RT_TLAS_LEAF
#define RT_TLAS_LEAF 4                                               // models per TLAS leaf.  Box tests per ray segment counted on the interpreter (tree + per-model, 500 instanced
                                                                     // models): leaf 1: 105.0, 2: 91.3, 4: 85.9, 8: 91.8
#endif
#ifndef RT_TLAS_SAH_DEPTH
#define RT_TLAS_SAH_DEPTH 10                                         // levels split by the surface-area heuristic; below: median (depth <= 10 + 11 < RT_TLAS_STACK)
#endif
    static_assert(SplitTreeStackBound(RT_TLAS_MAX_MODELS, RT_TLAS_SAH_DEPTH) <= RT_TLAS_STACK, "the TLAS walk's stack must hold the deepest TLAS");
    static constexpr int TLAS_AUTO_THRESHOLD = 128;                 // below it the linear test of every model box is cheaper than the TLAS walk

    // mode: 0 = off, 1 = on whenever it is possible, -1 = automatic (more than TLAS_AUTO_THRESHOLD models)
    static bool tlasWanted(int mode, int modelCount)
    {
        if (modelCount < 1 || modelCount > RT_TLAS_MAX_MODELS) return false;
        return mode > 0 || (mode < 0 && modelCount > TLAS_AUTO_THRESHOLD);
    }

    // Host only (no CUDA call).  A model with a singular worldToLocal carries an infinite box (buildModels); it
    // makes every TLAS box above it infinite, so it is always marked — conservative, like the linear test.
    // A TLAS box must reject a ray only where WorldBoxOutOfReach also rejects each model box below it.  Two kinds of box break the
    // plain union (buildModels never makes either, its padding is positive and finite): a flat box, whose slab WorldBoxOutOfReach
    // ignores for a ray lying in its plane (both slab distances 0 x inf = NaN), and a NaN bound, which leaves that slab to the other
    // bound alone or, for a ray in that bound's plane, ignores it.  The tree sees a flat box one ulp wider on each side and an axis with
    // a NaN bound as unbounded.
    static void planTlas(const std::vector<DevModel>& dm, int modelCount, std::vector<NodePair>& pairsOut, std::vector<int>& order, int& rootStart, int& rootCount)
    {
        const size_t n = (size_t)modelCount;
        std::vector<float> lo(3 * n), hi(3 * n), cen(3 * n);
        for (size_t i = 0; i < n; i++)
        {
            const float bmin[3] = {dm[i].wmin[0], dm[i].wmin[1], dm[i].wmin[2]}, bmax[3] = {dm[i].wmaxx, dm[i].wmaxy, dm[i].wmaxz};
            for (int a = 0; a < 3; a++)
            {
                float l = bmin[a], h = bmax[a];
                if (std::isnan(l) || std::isnan(h)) { l = -INFINITY; h = INFINITY; }
                else if (l == h && std::isfinite(l)) { l = std::nextafterf(l, -INFINITY); h = std::nextafterf(h, INFINITY); }
                lo[3 * i + a] = l; hi[3 * i + a] = h;
                const float c = 0.5f * bmin[a] + 0.5f * bmax[a];
                cen[3 * i + a] = std::isfinite(c) ? c : 0.0f;
            }
        }
        BuildMedianSplitPairs(lo, hi, cen, n, RT_TLAS_LEAF, order, pairsOut, rootStart, rootCount, RT_TLAS_SAH_DEPTH);
    }

    cudaError_t buildTlas(const std::vector<DevModel>& dm, int modelCount, int mode, cudaStream_t stream)
    {
        tlas = 0;
        if (!tlasWanted(mode, modelCount)) return cudaSuccess;
        std::vector<NodePair> pairsOut; std::vector<int> order;
        planTlas(dm, modelCount, pairsOut, order, tlasRootStart, tlasRootCount);
        cudaError_t e;
        if ((e = tlasPairs.ensure(std::max<size_t>(pairsOut.size(), 1))) != cudaSuccess) return e;
        if ((e = tlasLeaves.ensure(order.size())) != cudaSuccess) return e;
        if ((e = stageTlasPairs.acquire(pairsOut.size())) != cudaSuccess) return e;
        if ((e = stageTlasLeaves.acquire(order.size())) != cudaSuccess) return e;
        if (!pairsOut.empty()) memcpy(stageTlasPairs.p, pairsOut.data(), pairsOut.size() * sizeof(NodePair));
        memcpy(stageTlasLeaves.p, order.data(), order.size() * sizeof(int));
        if (!pairsOut.empty() && (e = cudaMemcpyAsync(tlasPairs.p, stageTlasPairs.p, pairsOut.size() * sizeof(NodePair), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(tlasLeaves.p, stageTlasLeaves.p, order.size() * sizeof(int), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = stageTlasPairs.commit(stream)) != cudaSuccess || (e = stageTlasLeaves.commit(stream)) != cudaSuccess) return e;
        tlas = 1;
        return cudaSuccess;
    }

    // Region of ray origins the padding of the current model boxes is valid for (see buildModels); models are rebuilt when the
    // camera or the geometry leaves it.
    float modelBoundLo[3] = {0, 0, 0}, modelBoundHi[3] = {0, 0, 0};
    bool modelBoundValid = false;
    bool modelBoundCovers(const float lo[3], const float hi[3]) const
    {
        if (!modelBoundValid) return false;
        for (int a = 0; a < 3; a++) if (!(lo[a] >= modelBoundLo[a] && hi[a] <= modelBoundHi[a])) return false;
        return true;
    }

    // Where a model's geometry is, as far as rays are concerned: the ray test only uses worldToLocal (HL:351-352) and a hit lies at
    // rayPos + rayDir * dst with dst found in the model's space, i.e. at inverse(worldToLocal) x (point of the mesh) — whatever
    // localToWorld says (it only turns normals, HL:367-368).  World box of the eight corners of the mesh's geometry box (MeshRoot::geo — the root's child boxes, not the root node's own bounds, which the
    // reference never reads) through that inverse (double);
    // false when worldToLocal is singular or not finite (nothing can be said about such a model).
    static bool worldBoxOfModel(const RtModel& m, const MeshRoot& root, double lo[3], double hi[3])
    {
        if (!root.geoValid) return false;
        const float* W = m.worldToLocal;                              // column-major 4x4, affine: x_local = A x_world + t
        const double A[3][3] = {{W[0], W[4], W[8]}, {W[1], W[5], W[9]}, {W[2], W[6], W[10]}}, t[3] = {W[12], W[13], W[14]};
        const double c00 = A[1][1] * A[2][2] - A[1][2] * A[2][1], c01 = A[1][2] * A[2][0] - A[1][0] * A[2][2], c02 = A[1][0] * A[2][1] - A[1][1] * A[2][0];
        const double det = A[0][0] * c00 + A[0][1] * c01 + A[0][2] * c02;
        double scale = 0;
        for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) scale = std::max(scale, std::fabs(A[r][c]));
        if (!(std::fabs(det) > 1e-12 * scale * scale * scale) || !std::isfinite(det)) return false;
        const double inv[3][3] = {
            {c00 / det, (A[0][2] * A[2][1] - A[0][1] * A[2][2]) / det, (A[0][1] * A[1][2] - A[0][2] * A[1][1]) / det},
            {c01 / det, (A[0][0] * A[2][2] - A[0][2] * A[2][0]) / det, (A[0][2] * A[1][0] - A[0][0] * A[1][2]) / det},
            {c02 / det, (A[0][1] * A[2][0] - A[0][0] * A[2][1]) / det, (A[0][0] * A[1][1] - A[0][1] * A[1][0]) / det}};
        for (int a = 0; a < 3; a++) { lo[a] = INFINITY; hi[a] = -INFINITY; }
        for (int k = 0; k < 8; k++)
        {
            const double v[3] = {(k & 1 ? root.geoHi[0] : root.geoLo[0]) - t[0], (k & 2 ? root.geoHi[1] : root.geoLo[1]) - t[1],
                                 (k & 4 ? root.geoHi[2] : root.geoLo[2]) - t[2]};
            for (int a = 0; a < 3; a++)
            {
                const double w = inv[a][0] * v[0] + inv[a][1] * v[1] + inv[a][2] * v[2];
                if (!std::isfinite(w) || std::fabs(w) > 1e30) return false;
                lo[a] = std::min(lo[a], w); hi[a] = std::max(hi[a], w);
            }
        }
        return true;
    }

    // originLo / originHi: a box containing every possible ray origin (camera with its defocus disc, all geometry; non-finite when
    // some model could not be placed).  The padding of the world boxes has three parts: 1e-4 of the box's own size and position,
    // 1e-5, and 2e-5 of the largest coordinate R in the origin box (RT_ORIGIN_PAD_SCALE).  The last one covers the arithmetic of a
    // ray that starts far away: the reference transforms the origin into the model's space and runs Moeller-Trumbore there, which
    // blurs where a ray "passes" by a few ulp(R) (the cross product of the origin offset with the direction cancels
    // catastrophically), and the slab test on the world box has its own few ulp(R); a hit the reference computes can lie that far
    // outside the exact geometry.  (Found with 1,500 two-centimetre models seen from 20,000 units away: without this part 3 pixels
    // of 36,864 differed from the oracle.)  If ray origins cannot be bounded, no model is skipped at all (every box is infinite).
    cudaError_t buildModels(const std::vector<RtModel>& mdl, const std::vector<RtNode>& nodes, int modelCount, cudaStream_t stream, int tlasMode,
                            const float originLo[3], const float originHi[3])
    {
        std::vector<DevModel> out(std::max(modelCount, 1));
        memset(out.data(), 0, out.size() * sizeof(DevModel));
        for (int a = 0; a < 3; a++) { modelBoundLo[a] = originLo[a]; modelBoundHi[a] = originHi[a]; }
        modelBoundValid = true;
        const double originPad = originPadOf(originLo, originHi);       // infinite when the origins are unbounded
        for (int i = 0; i < modelCount; i++)
        {
            DevModel d; memset(&d, 0, sizeof(d));
            for (int r = 0; r < 3; r++) for (int c = 0; c < 4; c++)
            {
                d.w2l[r * 4 + c] = mdl[i].worldToLocal[c * 4 + r];
                d.l2w[r * 4 + c] = mdl[i].localToWorld[c * 4 + r];
            }
            const MeshRoot& r = roots[std::make_pair(mdl[i].nodeOffset, mdl[i].triOffset)];
            d.rootStart = r.rootStart; d.rootCount = r.rootCount;
            d.cullBackface = mdl[i].material.flag != RT_MATERIAL_GLASS;       // HL:355
            d.matIndex = i;
            {
                double lo[3], hi[3];
                const bool placed = worldBoxOfModel(mdl[i], r, lo, hi);
                float bmin[3], bmax[3];
                paddedModelBox(placed, lo, hi, originPad, bmin, bmax);
                d.wmin[0] = bmin[0]; d.wmin[1] = bmin[1]; d.wmin[2] = bmin[2]; d.wmaxx = bmax[0]; d.wmaxy = bmax[1]; d.wmaxz = bmax[2];
            }
            out[i] = d;
        }
        cudaError_t e;
        if ((e = models.ensure(out.size())) != cudaSuccess) return e;
        if ((e = stageModels.acquire(out.size())) != cudaSuccess) return e;
        memcpy(stageModels.p, out.data(), out.size() * sizeof(DevModel));
        if ((e = cudaMemcpyAsync(models.p, stageModels.p, out.size() * sizeof(DevModel), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = stageModels.commit(stream)) != cudaSuccess) return e;
        return buildTlas(out, modelCount, tlasMode, stream);
    }

    // ---- spheres ------------------------------------------------------------------------------------------------------------
    RBuf<NodePair> sphPairs; RBuf<DevSphere> sphLeaves;
    int sphBvh = 0, sphRootStart = 0, sphRootCount = 0;
    float sphBoundLo[3] = {0, 0, 0}, sphBoundHi[3] = {0, 0, 0};     // region of ray origins the current padding is valid for
    static constexpr size_t SPHERE_BVH_THRESHOLD = 64;               // below this a linear scan is cheaper
#ifndef RT_SPHERE_LEAF
#define RT_SPHERE_LEAF 4                                              // spheres per leaf of the accelerator
#endif
#ifndef RT_SPHERE_SAH_DEPTH
#define RT_SPHERE_SAH_DEPTH 0                                        // top levels of the sphere tree by the surface-area sweep (see BuildMedianSplitPairs; 20 by default since round 2, rt_devmath.cuh); 0 = the measured median tree
#endif

    // Levels of the sphere tree split by the surface-area sweep for n spheres: RT_SPHERE_SAH_DEPTH, fewer where the deepest tree would
    // not fit TraverseSpheres' stack (beyond 2^27 spheres; a push that does not fit would lose a subtree).
    static int sphereSahDepth(long long n)
    {
        const int room = RT_SPHERE_STACK - SplitTreeStackBound(n, 0);
        return room < RT_SPHERE_SAH_DEPTH ? (room > 0 ? room : 0) : RT_SPHERE_SAH_DEPTH;
    }

    // Host only (no CUDA call): the accelerator's tree over the padded boxes of n spheres; order = sphere indices in leaf order.
    static void planSpheres(const RtSphere* sp, size_t n, const float originLo[3], const float originHi[3], std::vector<int>& order,
                            std::vector<NodePair>& pairsOut, int& rootStart, int& rootCount)
    {
        std::vector<float> lo(3 * n), hi(3 * n), cen(3 * n);
        for (size_t i = 0; i < n; i++)
        {
            paddedSphereBox(sp[i].centre, sp[i].radius, originLo, originHi, &lo[3 * i], &hi[3 * i]);
            for (int a = 0; a < 3; a++) cen[3 * i + a] = sp[i].centre[a];
        }
        BuildMedianSplitPairs(lo, hi, cen, n, RT_SPHERE_LEAF, order, pairsOut, rootStart, rootCount, sphereSahDepth((long long)n));
    }

    bool sphereBoundCovers(const float lo[3], const float hi[3]) const
    {
        for (int a = 0; a < 3; a++) if (lo[a] < sphBoundLo[a] || hi[a] > sphBoundHi[a]) return false;
        return true;
    }

    // originLo / originHi: a box containing every possible ray origin (camera, all geometry); only used for the BVH padding.
    cudaError_t buildSpheres(const std::vector<RtSphere>& sp, const float originLo[3], const float originHi[3], cudaStream_t stream)
    {
        std::vector<DevSphere> out(std::max<size_t>(sp.size(), 1));
        for (size_t i = 0; i < sp.size(); i++)
        {
            DevSphere d; memset(&d, 0, sizeof(d));
            d.cx = sp[i].centre[0]; d.cy = sp[i].centre[1]; d.cz = sp[i].centre[2]; d.radius = sp[i].radius;
            d.r2 = sphereR2(sp[i].radius);
            d.pad0 = sp[i].material.flag;                       // material flag, for sorting hits by kind without touching HBM
            d.pad1 = (int)i;
            out[i] = d;
        }
        cudaError_t e;
        if ((e = spheres.ensure(out.size())) != cudaSuccess) return e;
        if ((e = stageSpheres.acquire(out.size())) != cudaSuccess) return e;
        memcpy(stageSpheres.p, out.data(), out.size() * sizeof(DevSphere));
        if ((e = cudaMemcpyAsync(spheres.p, stageSpheres.p, out.size() * sizeof(DevSphere), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = stageSpheres.commit(stream)) != cudaSuccess) return e;
        sphBvh = 0;
        if (sp.size() <= SPHERE_BVH_THRESHOLD) return cudaSuccess;

        // ---- BVH over padded sphere boxes (see TraverseSpheres in rt_device.cuh for the exactness argument) ----
        // padding of sphere i: paddedSphereBox
        for (int a = 0; a < 3; a++) { sphBoundLo[a] = originLo[a]; sphBoundHi[a] = originHi[a]; }
        const size_t n = sp.size();
        // surface-area splits at the top, median splits below, leaves of RT_SPHERE_LEAF spheres; pairs emitted parent-before-children
        std::vector<int> order;
        std::vector<NodePair> pairsOut;
        planSpheres(sp.data(), n, originLo, originHi, order, pairsOut, sphRootStart, sphRootCount);
        std::vector<DevSphere> leaves(n);
        for (size_t k = 0; k < n; k++) leaves[k] = out[order[k]];
        if ((e = sphPairs.ensure(std::max<size_t>(pairsOut.size(), 1))) != cudaSuccess) return e;
        if ((e = sphLeaves.ensure(n)) != cudaSuccess) return e;
        if (!pairsOut.empty() && (e = cudaMemcpyAsync(sphPairs.p, pairsOut.data(), pairsOut.size() * sizeof(NodePair), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = cudaMemcpyAsync(sphLeaves.p, leaves.data(), n * sizeof(DevSphere), cudaMemcpyHostToDevice, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
        sphBvh = 1;
        return cudaSuccess;
    }
};

// ---- multi-GPU tile staging --------------------------------------------------------------------------------------------
// TileSend layout: [rowsPerRank rows of FrameRender | rowsPerRank rows of AccumulatedRender], rows in ascending
// global y of the bands this rank owns (band b belongs to rank b % world); ranks owning fewer rows pad.

__device__ __forceinline__ int owned_row_to_y(int r, int rank, int world, int bandRows)
{
    return ((r / bandRows) * world + rank) * bandRows + (r % bandRows);
}

__global__ void k_pack_tile(const float4* __restrict__ frame, const float4* __restrict__ accum, float4* __restrict__ send,
                            int W, int H, int rank, int world, int bandRows, int rowsPerRank)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    if (x >= W) return;
    const int y = owned_row_to_y(r, rank, world, bandRows);
    const size_t dst = (size_t)r * W + x;
    const size_t half = (size_t)rowsPerRank * W;
    if (y < H) { send[dst] = frame[(size_t)y * W + x]; send[half + dst] = accum[(size_t)y * W + x]; }
    else { send[dst] = make_float4(0, 0, 0, 0); send[half + dst] = make_float4(0, 0, 0, 0); }
}

__global__ void k_unpack_tiles(const float4* __restrict__ recv, float4* __restrict__ frame, float4* __restrict__ accum,
                               int W, int H, int world, int bandRows, int rowsPerRank)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y;
    const int rank = blockIdx.z;
    if (x >= W) return;
    const int y = owned_row_to_y(r, rank, world, bandRows);
    if (y >= H) return;
    const size_t half = (size_t)rowsPerRank * W;
    const float4* src = recv + (size_t)rank * 2 * half;
    frame[(size_t)y * W + x] = src[(size_t)r * W + x];
    accum[(size_t)y * W + x] = src[half + (size_t)r * W + x];
}

__global__ void k_display(const float4* __restrict__ tex, uchar4* __restrict__ out, size_t n, float frame)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 t = tex[i];
    out[i] = make_uchar4((unsigned char)DisplayEncode(t.x / frame), (unsigned char)DisplayEncode(t.y / frame),
                         (unsigned char)DisplayEncode(t.z / frame), (unsigned char)DisplayEncode(t.w / frame));
}

// Heat map of the per-pixel counters (rtDisplayPixelStats; the encode is pinned in include/rt_b200.h so that the oracle restates it
// bit for bit).  The clamp is written as comparisons: t > 1 is red, every other t lies in [0, 1] and needs no saturation.
__global__ void k_pixel_stats_display(const RtPixelStats* __restrict__ st, uchar4* __restrict__ out, size_t n, int visMode, float scale)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const RtPixelStats s = st[i];
    if (s.rays == 0u) { out[i] = make_uchar4(0, 0, 0, 255); return; }
    const unsigned int count = visMode == 1 ? s.boxTests : visMode == 2 ? s.triTests : s.sphereTests + s.sphereBoxTests;
    const float v = visMode == 4 ? __uint2float_rn(s.rays) : __uint2float_rn(count) / __uint2float_rn(s.rays);
    const float t = v / scale;
    if (t > 1.0f) { out[i] = make_uchar4(255, 0, 0, 255); return; }
    const unsigned char g = (unsigned char)__float2uint_rz(t * 255.0f + 0.5f);
    out[i] = make_uchar4(g, g, g, 255);
}

inline void launch_pack_tile(const float4* frame, const float4* accum, float4* send, int W, int H, int rank, int world, int bandRows, int rowsPerRank, cudaStream_t s)
{
    dim3 grid((W + 255) / 256, rowsPerRank, 1);
    RT_LAUNCH(grid, 256, 0, s, k_pack_tile, frame, accum, send, W, H, rank, world, bandRows, rowsPerRank);
}
inline void launch_unpack_tiles(const float4* recv, float4* frame, float4* accum, int W, int H, int world, int bandRows, int rowsPerRank, cudaStream_t s)
{
    dim3 grid((W + 255) / 256, rowsPerRank, world);
    RT_LAUNCH(grid, 256, 0, s, k_unpack_tiles, recv, frame, accum, W, H, world, bandRows, rowsPerRank);
}

} // namespace rtd
