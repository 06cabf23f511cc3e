// BVH.cpp — see BVH.h.  Splitting rules follow Assets/Scripts/Types/BVH.cs:26-318 of the reference.
#include "BVH.h"

#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <stdexcept>
#include <thread>

namespace Seb {

int BVH::BuildThreads = 0;

namespace {

constexpr int kParallelMinTris = 16384;      // below this a subtree is built by one thread

struct Box
{
    float lo[3], hi[3];
    Box() { for (int a = 0; a < 3; a++) { lo[a] = FLT_MAX; hi[a] = -FLT_MAX; } }    // float.MaxValue / float.MinValue (BVH.cs:37-42)
    template <class T> void grow(const T& t)
    {
        if (t.minX < lo[0]) lo[0] = t.minX;
        if (t.minY < lo[1]) lo[1] = t.minY;
        if (t.minZ < lo[2]) lo[2] = t.minZ;
        if (t.maxX > hi[0]) hi[0] = t.maxX;
        if (t.maxY > hi[1]) hi[1] = t.maxY;
        if (t.maxZ > hi[2]) hi[2] = t.maxZ;
    }
};

inline float min3(float a, float b, float c) { return a < b ? (a < c ? a : c) : (b < c ? b : c); }   // BVH.cs:488-490
inline float max3(float a, float b, float c) { return a > b ? (a > c ? a : c) : (b > c ? b : c); }   // BVH.cs:491-493

inline RtNode makeNode(const Box& b, int start, int count)
{
    RtNode n;
    for (int a = 0; a < 3; a++) { n.boundsMin[a] = b.lo[a]; n.boundsMax[a] = b.hi[a]; }
    n.startIndex = start; n.triangleCount = count;
    return n;
}

} // namespace

static void mergeStats(BVH::BuildStats& a, const BVH::BuildStats& b)
{
    a.TriangleCount += b.TriangleCount; a.TotalNodeCount += b.TotalNodeCount; a.LeafNodeCount += b.LeafNodeCount; a.LeafDepthSum += b.LeafDepthSum;
    if (b.LeafDepthMax > a.LeafDepthMax) a.LeafDepthMax = b.LeafDepthMax;
    if (b.LeafDepthMin < a.LeafDepthMin) a.LeafDepthMin = b.LeafDepthMin;
    if (b.LeafMaxTriCount > a.LeafMaxTriCount) a.LeafMaxTriCount = b.LeafMaxTriCount;
    if (b.LeafMinTriCount < a.LeafMinTriCount) a.LeafMinTriCount = b.LeafMinTriCount;
}

void BVH::BuildStats::RecordNode(int depth, bool isLeaf, int triCount)
{
    TotalNodeCount++;
    if (!isLeaf) return;
    LeafNodeCount++;
    LeafDepthSum += depth;
    if (depth < LeafDepthMin) LeafDepthMin = depth;
    if (depth > LeafDepthMax) LeafDepthMax = depth;
    TriangleCount += triCount;
    if (triCount > LeafMaxTriCount) LeafMaxTriCount = triCount;
    if (triCount < LeafMinTriCount) LeafMinTriCount = triCount;
}

std::string BVH::BuildStats::ToString() const
{
    char buf[512];
    const char* q = quality == Quality::Low ? "Low" : quality == Quality::High ? "High" : "Disabled";
    snprintf(buf, sizeof(buf),
             "Time (BVH): %d ms (quality = %s)\nTriangles: %d\nNode Count: %d\nLeaf Count: %d\nLeaf Depth:\n - Min: %d\n - Max: %d\n - Mean: %.4g\n"
             "Leaf Tris:\n - Min: %d\n - Max: %d\n - Mean: %.4g\n",
             TimeMs, q, TriangleCount, TotalNodeCount, LeafNodeCount, LeafDepthMin, LeafDepthMax,
             LeafNodeCount ? LeafDepthSum / (float)LeafNodeCount : 0.0f, LeafMinTriCount, LeafMaxTriCount,
             LeafNodeCount ? TriangleCount / (float)LeafNodeCount : 0.0f);
    return buf;
}

BVH::BVH(const Vector3* verts, int vertCount, const int* indices, int indexCount, const Vector3* normals, Quality q)
    : quality(q)
{
    const auto t0 = std::chrono::steady_clock::now();
    stats.quality = q;
    if (indexCount <= 0 || indexCount % 3 != 0) throw std::invalid_argument("BVH: index count must be a positive multiple of 3");
    for (int i = 0; i < indexCount; i++)
        if (indices[i] < 0 || indices[i] >= vertCount) throw std::invalid_argument("BVH: vertex index out of range");

    const int triCount = indexCount / 3;
    int threads = BuildThreads > 0 ? BuildThreads : (int)std::thread::hardware_concurrency();
    if (threads < 1) threads = 1;
    if (threads > 128) threads = 128;
    if (triCount < kParallelMinTris) threads = 1;
    // run f(t, lo, hi) on `threads` slices of [0, triCount)
    auto parallelSlices = [&](auto&& f)
    {
        std::vector<std::thread> pool;
        for (int t = 1; t < threads; t++) pool.emplace_back([&, t]() { f(t, (int)((long long)triCount * t / threads), (int)((long long)triCount * (t + 1) / threads)); });
        f(0, 0, (int)((long long)triCount / threads));
        for (auto& th : pool) th.join();
    };

    buildTris.resize(triCount);
    std::vector<Box> sliceBox(threads);
    parallelSlices([&](int t, int lo, int hi)
    {
        for (int k = lo; k < hi; k++)                               // BVH.cs:44-59
        {
            const int i = 3 * k;
            const Vector3 a = verts[indices[i]], b = verts[indices[i + 1]], c = verts[indices[i + 2]];
            BuildTri tr;
            tr.cx = (a.x + b.x + c.x) / 3; tr.cy = (a.y + b.y + c.y) / 3; tr.cz = (a.z + b.z + c.z) / 3;
            tr.minX = min3(a.x, b.x, c.x); tr.minY = min3(a.y, b.y, c.y); tr.minZ = min3(a.z, b.z, c.z);
            tr.maxX = max3(a.x, b.x, c.x); tr.maxY = max3(a.y, b.y, c.y); tr.maxZ = max3(a.z, b.z, c.z);
            tr.index = i;
            buildTris[k] = tr;
            sliceBox[t].grow(tr);
        }
    });
    Box all;
    for (const Box& b : sliceBox) for (int a = 0; a < 3; a++) { if (b.lo[a] < all.lo[a]) all.lo[a] = b.lo[a]; if (b.hi[a] > all.hi[a]) all.hi[a] = b.hi[a]; }

    Nodes.reserve(256);
    AddNode(makeNode(all, -1, -1));                               // BVH.cs:61
    if (quality == Quality::Disabled) { Nodes[0].startIndex = 0; Nodes[0].triangleCount = triCount; }
    else if (threads == 1 || triCount < kParallelMinTris) Split(Nodes, stats, 0, 0, triCount, 0);
    else
    {
        // the same recursion, its independent subtrees built by different threads and concatenated in the reference's order
        Block blk;
        bool rootInner = false;
        RtNode root = BuildBlock(Nodes[0], 0, triCount, 0, blk, threads, rootInner);
        if (rootInner) root.startIndex = 1;                               // B(root) starts right after the root
        for (size_t k = 0; k < blk.nodes.size(); k++) if (blk.inner[k]) blk.nodes[k].startIndex += 1;
        Nodes[0] = root;
        Nodes.insert(Nodes.end(), blk.nodes.begin(), blk.nodes.end());
        mergeStats(stats, blk.stats);
    }

    Triangles.resize(triCount);                                   // BVH.cs:69-80: leaf order
    parallelSlices([&](int, int lo, int hi)
    {
    for (int i = lo; i < hi; i++)
    {
        const int base = buildTris[i].index;
        RtTriangle& o = Triangles[i];
        const Vector3* p[3] = {&verts[indices[base]], &verts[indices[base + 1]], &verts[indices[base + 2]]};
        const Vector3* n[3] = {&normals[indices[base]], &normals[indices[base + 1]], &normals[indices[base + 2]]};
        o.posA[0] = p[0]->x; o.posA[1] = p[0]->y; o.posA[2] = p[0]->z;
        o.posB[0] = p[1]->x; o.posB[1] = p[1]->y; o.posB[2] = p[1]->z;
        o.posC[0] = p[2]->x; o.posC[1] = p[2]->y; o.posC[2] = p[2]->z;
        o.normA[0] = n[0]->x; o.normA[1] = n[0]->y; o.normA[2] = n[0]->z;
        o.normB[0] = n[1]->x; o.normB[1] = n[1]->y; o.normB[2] = n[1]->z;
        o.normC[0] = n[2]->x; o.normC[1] = n[2]->y; o.normC[2] = n[2]->z;
    }
    });
    std::vector<BuildTri>().swap(buildTris);
    stats.TimeMs = (int)std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::steady_clock::now() - t0).count();
}

int BVH::AddNode(const RtNode& n) { Nodes.push_back(n); return (int)Nodes.size() - 1; }

float BVH::NodeCost(float x, float y, float z, int numTriangles)  // BVH.cs:313-318
{
    if (numTriangles == 0) return 0;
    const float area = x * y + x * z + y * z;
    return area * numTriangles;
}

float BVH::EvaluateSplit(int splitAxis, float splitPos, int start, int count) const   // BVH.cs:253-311
{
    Box left, right;
    int numOnLeft = 0, numOnRight = 0;
    for (int i = start; i < start + count; i++)
    {
        const BuildTri& t = buildTris[i];
        const float c = splitAxis == 0 ? t.cx : splitAxis == 1 ? t.cy : t.cz;
        if (c < splitPos) { left.grow(t); numOnLeft++; }
        else { right.grow(t); numOnRight++; }
    }
    const float costA = NodeCost(left.hi[0] - left.lo[0], left.hi[1] - left.lo[1], left.hi[2] - left.lo[2], numOnLeft);
    const float costB = NodeCost(right.hi[0] - right.lo[0], right.hi[1] - right.lo[1], right.hi[2] - right.lo[2], numOnRight);
    return costA + costB;
}

namespace {
struct CandidateAcc { Box left, right; int numOnLeft = 0, numOnRight = 0; };
}

BVH::SplitChoice BVH::ChooseSplit(const RtNode& node, int start, int count, int threads) const     // BVH.cs:183-250
{
    if (count <= 1) return SplitChoice{0, 0.0f, INFINITY};
    const float size[3] = {node.boundsMax[0] - node.boundsMin[0], node.boundsMax[1] - node.boundsMin[1], node.boundsMax[2] - node.boundsMin[2]};

    if (quality == Quality::Low)
    {
        const int axis = size[0] > size[1] && size[0] > size[2] ? 0 : size[1] > size[2] ? 1 : 2;
        const float pos = node.boundsMin[axis] + size[axis] * 0.5f;
        return SplitChoice{axis, pos, EvaluateSplit(axis, pos, start, count)};
    }

    SplitChoice best{0, 0.0f, FLT_MAX};
    const int maxSplitTests = count < 10 ? 3 : 5;
    float maxAxis = size[0];                                      // Mathf.Max(sizeX, sizeY, sizeZ)
    if (size[1] > maxAxis) maxAxis = size[1];
    if (size[2] > maxAxis) maxAxis = size[2];

    int candAxis[15]; float candPos[15]; int numCand = 0;
    for (int axis = 0; axis < 3; axis++)
    {
        const float ratio = size[axis] / maxAxis * maxSplitTests;
        // Mathf.CeilToInt; a NaN ratio (degenerate node, 0/0) ends up at the lower clamp like C#'s (int)NaN = int.MinValue
        int numSplitTests = std::isnan(ratio) ? 1 : (int)std::ceil((double)ratio);
        if (numSplitTests < 1) numSplitTests = 1;
        if (numSplitTests > maxSplitTests) numSplitTests = maxSplitTests;
        for (int i = 0; i < numSplitTests; i++)
        {
            const float splitT = (i + 1) / (numSplitTests + 1.0f);
            candAxis[numCand] = axis; candPos[numCand] = node.boundsMin[axis] + size[axis] * splitT; numCand++;
        }
    }
    if (threads <= 1 || count < kParallelMinTris)
    {
        for (int c = 0; c < numCand; c++)
        {
            const float cost = EvaluateSplit(candAxis[c], candPos[c], start, count);
            if (cost < best.cost) { best.cost = cost; best.pos = candPos[c]; best.axis = candAxis[c]; }
        }
        return best;
    }
    // large node: every thread takes a slice of the triangles and evaluates all candidates on it in one pass; boxes merge by
    // min / max and counts by sum, which are exact in any order, so the costs are the serial EvaluateSplit's bit for bit
    std::vector<std::vector<CandidateAcc>> part(threads, std::vector<CandidateAcc>(numCand));
    auto slice = [&](int t)
    {
        const int lo = start + (int)((long long)count * t / threads), hi = start + (int)((long long)count * (t + 1) / threads);
        std::vector<CandidateAcc>& acc = part[t];
        for (int i = lo; i < hi; i++)
        {
            const BuildTri& tri = buildTris[i];
            for (int c = 0; c < numCand; c++)
            {
                const float centre = candAxis[c] == 0 ? tri.cx : candAxis[c] == 1 ? tri.cy : tri.cz;
                if (centre < candPos[c]) { acc[c].left.grow(tri); acc[c].numOnLeft++; }
                else { acc[c].right.grow(tri); acc[c].numOnRight++; }
            }
        }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < threads; t++) pool.emplace_back(slice, t);
    slice(0);
    for (auto& th : pool) th.join();
    for (int c = 0; c < numCand; c++)
    {
        CandidateAcc total;
        for (int t = 0; t < threads; t++)
        {
            const CandidateAcc& a = part[t][c];
            for (int k = 0; k < 3; k++)
            {
                if (a.left.lo[k] < total.left.lo[k]) total.left.lo[k] = a.left.lo[k];
                if (a.left.hi[k] > total.left.hi[k]) total.left.hi[k] = a.left.hi[k];
                if (a.right.lo[k] < total.right.lo[k]) total.right.lo[k] = a.right.lo[k];
                if (a.right.hi[k] > total.right.hi[k]) total.right.hi[k] = a.right.hi[k];
            }
            total.numOnLeft += a.numOnLeft; total.numOnRight += a.numOnRight;
        }
        const float costA = NodeCost(total.left.hi[0] - total.left.lo[0], total.left.hi[1] - total.left.lo[1], total.left.hi[2] - total.left.lo[2], total.numOnLeft);
        const float costB = NodeCost(total.right.hi[0] - total.right.lo[0], total.right.hi[1] - total.right.lo[1], total.right.hi[2] - total.right.lo[2], total.numOnRight);
        const float cost = costA + costB;
        if (cost < best.cost) { best.cost = cost; best.pos = candPos[c]; best.axis = candAxis[c]; }
    }
    return best;
}

void BVH::Split(std::vector<RtNode>& Nodes, BuildStats& stats, int parentIndex, int triGlobalStart, int triNum, int depth, std::vector<char>* inner)   // BVH.cs:89-181
{
    const int MaxDepth = 32;
    const RtNode parent = Nodes[parentIndex];
    const float parentCost = NodeCost(parent.boundsMax[0] - parent.boundsMin[0], parent.boundsMax[1] - parent.boundsMin[1],
                                      parent.boundsMax[2] - parent.boundsMin[2], triNum);
    const SplitChoice split = ChooseSplit(parent, triGlobalStart, triNum);

    if (split.cost < parentCost && depth < MaxDepth)
    {
        Box left, right;
        int numOnLeft = 0;
        for (int i = triGlobalStart; i < triGlobalStart + triNum; i++)
        {
            const BuildTri t = buildTris[i];
            const float c = split.axis == 0 ? t.cx : split.axis == 1 ? t.cy : t.cz;
            if (c < split.pos)
            {
                left.grow(t);
                // swap into the left partition (BVH.cs:138-141)
                const BuildTri other = buildTris[triGlobalStart + numOnLeft];
                buildTris[triGlobalStart + numOnLeft] = t;
                buildTris[i] = other;
                numOnLeft++;
            }
            else right.grow(t);
        }
        const int numOnRight = triNum - numOnLeft;
        Nodes.push_back(makeNode(left, triGlobalStart, 0));
        const int childIndexLeft = (int)Nodes.size() - 1;
        Nodes.push_back(makeNode(right, triGlobalStart + numOnLeft, 0));
        const int childIndexRight = childIndexLeft + 1;
        Nodes[parentIndex].startIndex = childIndexLeft;
        if (inner) { inner->resize(Nodes.size(), 0); (*inner)[parentIndex] = 1; }
        stats.RecordNode(depth, false);
        Split(Nodes, stats, childIndexLeft, triGlobalStart, numOnLeft, depth + 1, inner);
        Split(Nodes, stats, childIndexRight, triGlobalStart + numOnLeft, numOnRight, depth + 1, inner);
    }
    else
    {
        Nodes[parentIndex].startIndex = triGlobalStart;
        Nodes[parentIndex].triangleCount = triNum;
        stats.RecordNode(depth, true, triNum);
    }
}

// The subtree below `node` (its triangles are buildTris[triGlobalStart .. +triNum)), built with up to `threads` threads.
// Takes exactly the decisions Split() takes — same ChooseSplit, same in-place partition — and returns the node with its leaf
// range or, for an inner node, startIndex = 0 (block-relative); blk receives B(node), isInner whether Split split the node.
// Only inner nodes' startIndex is a child index to rebase.  triangleCount cannot tell: an empty leaf (a split that put every
// triangle on one side, e.g. when every cost is inf) has triangleCount 0 like an inner node, and startIndex = its triangle start.
RtNode BVH::BuildBlock(RtNode node, int triGlobalStart, int triNum, int depth, Block& blk, int threads, bool& isInner)
{
    if (threads <= 1 || triNum < kParallelMinTris)
    {
        std::vector<RtNode> local;
        std::vector<char> localInner(1, 0);
        local.reserve((size_t)triNum / 2 + 16);
        local.push_back(node);
        Split(local, blk.stats, 0, triGlobalStart, triNum, depth, &localInner);
        node = local[0];
        isInner = localInner[0] != 0;
        blk.nodes.assign(local.begin() + 1, local.end());
        blk.inner.assign(localInner.begin() + 1, localInner.end());
        for (size_t k = 0; k < blk.nodes.size(); k++) if (blk.inner[k]) blk.nodes[k].startIndex -= 1;    // local index -> block-relative
        if (isInner) node.startIndex = 0;
        return node;
    }
    const int MaxDepth = 32;
    const float parentCost = NodeCost(node.boundsMax[0] - node.boundsMin[0], node.boundsMax[1] - node.boundsMin[1], node.boundsMax[2] - node.boundsMin[2], triNum);
    const SplitChoice split = ChooseSplit(node, triGlobalStart, triNum, threads);
    if (!(split.cost < parentCost && depth < MaxDepth))
    {
        node.startIndex = triGlobalStart; node.triangleCount = triNum;
        blk.stats.RecordNode(depth, true, triNum);
        isInner = false;
        return node;
    }
    Box left, right;
    int numOnLeft = 0;
    for (int i = triGlobalStart; i < triGlobalStart + triNum; i++)          // the reference's partition, sequential: its order is part of the result
    {
        const BuildTri t = buildTris[i];
        const float c = split.axis == 0 ? t.cx : split.axis == 1 ? t.cy : t.cz;
        if (c < split.pos)
        {
            left.grow(t);
            const BuildTri other = buildTris[triGlobalStart + numOnLeft];
            buildTris[triGlobalStart + numOnLeft] = t;
            buildTris[i] = other;
            numOnLeft++;
        }
        else right.grow(t);
    }
    const int numOnRight = triNum - numOnLeft;
    RtNode childL = makeNode(left, triGlobalStart, 0), childR = makeNode(right, triGlobalStart + numOnLeft, 0);
    blk.stats.RecordNode(depth, false);
    int threadsL = (int)((long long)threads * numOnLeft / triNum);
    if (threadsL < 1) threadsL = 1;
    if (threadsL > threads - 1) threadsL = threads - 1;
    Block bl, br;
    bool innerL = false, innerR = false;
    std::thread worker([&]() { childL = BuildBlock(childL, triGlobalStart, numOnLeft, depth + 1, bl, threadsL, innerL); });
    childR = BuildBlock(childR, triGlobalStart + numOnLeft, numOnRight, depth + 1, br, threads - threadsL, innerR);
    worker.join();
    // B(node) = [L, R] + B(L) + B(R)
    const int offL = 2, offR = 2 + (int)bl.nodes.size();
    if (innerL) childL.startIndex = offL;
    if (innerR) childR.startIndex = offR;
    blk.nodes.reserve(2 + bl.nodes.size() + br.nodes.size());
    blk.inner.reserve(2 + bl.inner.size() + br.inner.size());
    blk.nodes.push_back(childL); blk.nodes.push_back(childR);
    blk.inner.push_back(innerL); blk.inner.push_back(innerR);
    for (size_t k = 0; k < bl.nodes.size(); k++) { if (bl.inner[k]) bl.nodes[k].startIndex += offL; blk.nodes.push_back(bl.nodes[k]); blk.inner.push_back(bl.inner[k]); }
    for (size_t k = 0; k < br.nodes.size(); k++) { if (br.inner[k]) br.nodes[k].startIndex += offR; blk.nodes.push_back(br.nodes[k]); blk.inner.push_back(br.inner[k]); }
    mergeStats(blk.stats, bl.stats); mergeStats(blk.stats, br.stats);
    node.startIndex = 0;
    isInner = true;
    return node;
}

} // namespace Seb
