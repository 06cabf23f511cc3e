// BVH.h — host-side BVH builder producing the Nodes / Triangles buffers the kernel consumes.
//
// Mirrors the public surface of the reference's C# class Seb.AccelerationStructures.BVH
// (Assets/Scripts/Types/BVH.cs:9-87: Quality enum, Triangles, Nodes, stats, constructor arguments) so the
// host code above the C-ABI reads like the reference's.  The build reproduces the reference's splitting
// rules (BVH.cs:89-318) — same candidate planes, same cost, same in-place partition, children allocated
// adjacently, left subtree first — so node order, leaf contents and triangle order are those the reference
// would upload.  All arithmetic is FP32 (built with -ffp-contract=off).
#pragma once
#include "rt_types.h"
#include <string>
#include <vector>

namespace Seb {

struct Vector3 { float x, y, z; };

class BVH
{
public:
    enum class Quality { Low = 0, High = 1, Disabled = 2 };      // BVH.cs:11-16

    struct BuildStats                                             // BVH.cs:519-576
    {
        int TimeMs = 0;
        int TriangleCount = 0;
        int TotalNodeCount = 0;
        int LeafNodeCount = 0;
        int LeafDepthMax = 0;
        int LeafDepthMin = 0x7fffffff;
        int LeafDepthSum = 0;
        int LeafMaxTriCount = 0;
        int LeafMinTriCount = 0x7fffffff;
        Quality quality = Quality::High;
        void RecordNode(int depth, bool isLeaf, int triCount = 0);
        std::string ToString() const;
    };

    std::vector<RtTriangle> Triangles;
    std::vector<RtNode> Nodes;
    BuildStats stats;

    // verts / normals: per-vertex arrays; indices: 3 per triangle (Unity Mesh.vertices / .triangles / .normals)
    BVH(const Vector3* verts, int vertCount, const int* indices, int indexCount, const Vector3* normals, Quality quality = Quality::High);

    // Host threads a build may use (0 = all hardware threads, 1 = the reference's single-threaded recursion).  The result does not
    // depend on it: the same nodes in the same order, the same triangle order, byte for byte (tests/test_host.py).
    static int BuildThreads;

private:
    struct BuildTri { float cx, cy, cz, minX, minY, minZ, maxX, maxY, maxZ; int index; };   // BVH.cs:459-496
    struct SplitChoice { int axis; float pos; float cost; };

    std::vector<BuildTri> buildTris;
    Quality quality;

    // B(n) of a node n: everything Split(n) appends to Nodes — [left child, right child] + B(left) + B(right) — with child
    // indices relative to the first entry of the block, so that independently built blocks concatenate by adding offsets.
    // inner[k] says whether nodes[k] was split (its startIndex is a child index) or is a leaf, empty leaves included.
    struct Block { std::vector<RtNode> nodes; std::vector<char> inner; BuildStats stats; };

    int  AddNode(const RtNode& n);
    // inner (optional): set to 1 at every node Split splits, grown with the node list
    void Split(std::vector<RtNode>& nodes, BuildStats& st, int parentIndex, int triGlobalStart, int triNum, int depth, std::vector<char>* inner = nullptr);
    RtNode BuildBlock(RtNode node, int triGlobalStart, int triNum, int depth, Block& blk, int threads, bool& isInner);
    SplitChoice ChooseSplit(const RtNode& node, int start, int count, int threads = 1) const;
    float EvaluateSplit(int splitAxis, float splitPos, int start, int count) const;
    static float NodeCost(float x, float y, float z, int numTriangles);
};

} // namespace Seb
