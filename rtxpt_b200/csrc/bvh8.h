// bvh8.h — compressed 8-wide BVH (CWBVH8) layout shared by the host builder and the device traversal.
//
// The reference has no acceleration-structure format to follow: BLAS/TLAS are opaque driver objects
// (Rtxpt/Sample.cpp:1061-1240, Rtxpt/SampleCommon/AccelerationStructureUtil.h:34-100).  This is the layout of
//   H. Ylitie, T. Karras, S. Laine, "Efficient Incoherent Ray Traversal on GPUs Through Compressed Wide BVHs", HPG 2017
// 80-byte nodes (5 x 16 B, one 128-bit load each) and 48-byte triangles (3 x 16 B).
//
// Node (80 B):
//   q0: p.x p.y p.z | ex ey ez imask          origin of the quantisation grid, per-axis exponent (biased, 2^(e-127)), internal-child mask
//   q1: childBase | triBase | meta[0..3] | meta[4..7]
//        meta[i] = 0                        empty slot
//        meta[i] = 0b001_11sss (0x38 | s)   internal child in slot s (s == i)
//        meta[i] = uuu_ooooo                leaf: ooooo = first triangle (offset from triBase, 0..23), uuu = unary count 001/011/111
//   q2: qlo.x[0..7] | qlo.y[0..7]
//   q3: qlo.z[0..7] | qhi.x[0..7]
//   q4: qhi.y[0..7] | qhi.z[0..7]
//   Slot s holds the child lying towards direction (s&4 ? +x : -x, s&2 ? +y : -y, s&1 ? +z : -z) so that visiting slots in the
//   order (s XOR octant) gives front-to-back traversal for every ray octant.
// Triangle (48 B): v0.xyz gid | v1.xyz subInstanceAndFlags | v2.xyz opacity-mask slot (0xFFFFFFFF: none; field `primitiveIndex` of BuildTriangle / Bvh8Tri)
//   gid  = global triangle id (instance order, geometry order, primitive order) — the tie-break key for equal-t hits
//   subInstanceAndFlags = subInstanceIndex | (alphaTested << 30) | (excludeFromNEE << 31)
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>
#include <vector>

namespace pt {

struct Bvh8Node { uint32_t w[20]; };        // 80 bytes
struct Bvh8Tri  { float v0[3]; uint32_t gid; float v1[3]; uint32_t subInstanceAndFlags; float v2[3]; uint32_t primitiveIndex; };   // 48 bytes

constexpr uint32_t kTriFlagAlphaTested = 1u << 30;
constexpr uint32_t kTriFlagExcludeFromNEE = 1u << 31;
constexpr uint32_t kTriSubInstanceMask = (1u << 30) - 1u;

struct BuildTriangle { float v0[3], v1[3], v2[3]; uint32_t gid, subInstanceAndFlags, primitiveIndex; };

struct Bvh8
{
    std::vector<Bvh8Node> nodes;    // breadth-first: the top of the tree is a prefix of the array (staged into shared memory by the kernels)
    std::vector<uint32_t> levelStart;   // nodes of depth d (root = 0) are [levelStart[d], levelStart[d + 1]): what a bottom-up refit walks, deepest level first (refit.cuh)
    std::vector<Bvh8Tri> tris;      // leaf order
    float sceneLo[3], sceneHi[3];
    double buildSeconds = 0;
    uint32_t maxDepth = 0;
};

// ---- quantisation frame, shared by the host builder and the device refit (refit.cuh) so that a refit of unmoved geometry reproduces the built nodes bit for bit ----
#if defined(__CUDACC__)
#define BVH8_HD __host__ __device__ inline
#else
#define BVH8_HD inline
#endif
// exponent of a node axis: the smallest e in [-126, 100] with ext / 2^e <= 255, found with exact operations only (traverse.cuh scales by a further 2^15 and by 1/|d| <= 1e20)
BVH8_HD int bvh8FrameExponent(double ext)
{
    if (!(ext > 0.0)) return -126;
    int k = 0; (void)frexp(ext, &k);                     // ext = m * 2^k, m in [0.5, 1)
    int e = k - 8;                                       // 255 < 2^8: ext / 2^(k-8) = m * 256 in [128, 256)
    if (e < -126) e = -126;
    if (e > 100) e = 100;
    while (e < 100 && ext / ldexp(1.0, e) > 255.0) e++;
    while (e > -126 && ext / ldexp(1.0, e - 1) <= 255.0) e--;
    return e;
}
// conservative 8-bit box of a child inside its parent's frame: floor / ceil in double, clamped to the grid
BVH8_HD void bvh8QuantizeChild(const float* nodeLo, const uint32_t* ebias, const float* childLo, const float* childHi, uint8_t* qlo, uint8_t* qhi)
{
    for (int a = 0; a < 3; a++)
    {
        const double scale = ldexp(1.0, int(ebias[a]) - 127);
        const double lo = floor((double(childLo[a]) - double(nodeLo[a])) / scale), hi = ceil((double(childHi[a]) - double(nodeLo[a])) / scale);
        qlo[a] = uint8_t(lo < 0.0 ? 0.0 : (lo > 255.0 ? 255.0 : lo)); qhi[a] = uint8_t(hi < 0.0 ? 0.0 : (hi > 255.0 ? 255.0 : hi));
    }
}

// ---- octant slot assignment and node encoding, shared by the host builder (bvh_builder.cpp) and the device builder (bvh_build.cuh) ----
// children (boxes in any order) -> slot of each: greedy maximum of dot(child centre - node centre, slot direction), first child / slot on ties
BVH8_HD void bvh8AssignSlots(const float* nodeLo, const float* nodeHi, int nChild, const float (*childLo)[3], const float (*childHi)[3], int* childInSlot)
{
    float nc[3]; for (int a = 0; a < 3; a++) nc[a] = 0.5f * (nodeLo[a] + nodeHi[a]);
    float cost[8][8];
    for (int i = 0; i < nChild; i++)
    {
        float d[3]; for (int a = 0; a < 3; a++) d[a] = 0.5f * (childLo[i][a] + childHi[i][a]) - nc[a];
        for (int s = 0; s < 8; s++) cost[i][s] = ((s & 4) ? d[0] : -d[0]) + ((s & 2) ? d[1] : -d[1]) + ((s & 1) ? d[2] : -d[2]);
    }
    int slotOf[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }; bool slotUsed[8] = { false, false, false, false, false, false, false, false }; bool childDone[8] = { false, false, false, false, false, false, false, false };
    for (int k = 0; k < nChild; k++)
    {
        float bestC = -3.0e38f; int bi = -1, bs = -1;
        for (int i = 0; i < nChild; i++) if (!childDone[i]) for (int s = 0; s < 8; s++) if (!slotUsed[s] && cost[i][s] > bestC) { bestC = cost[i][s]; bi = i; bs = s; }
        slotOf[bi] = bs; slotUsed[bs] = true; childDone[bi] = true;
    }
    for (int s = 0; s < 8; s++) childInSlot[s] = -1;
    for (int i = 0; i < nChild; i++) childInSlot[slotOf[i]] = i;
}
// one 80-byte node from its box, the boxes of the used slots (meta[s] != 0), the slot metadata and the child / triangle bases: quantisation frame and conservative child boxes
BVH8_HD void bvh8EncodeNode(const float* lo, const float* hi, const float (*slotLo)[3], const float (*slotHi)[3], const uint8_t* meta, uint32_t imask, uint32_t childBase, uint32_t triBase,
                            uint32_t* w)
{
    uint32_t ebias[3];
    for (int a = 0; a < 3; a++) ebias[a] = uint32_t(bvh8FrameExponent(double(hi[a]) - double(lo[a])) + 127);
    uint8_t q[6][8];
    for (int k = 0; k < 6; k++) for (int s = 0; s < 8; s++) q[k][s] = 0;
    for (int s = 0; s < 8; s++)
    {
        if (meta[s] == 0) continue;
        uint8_t ql[3], qh[3]; bvh8QuantizeChild(lo, ebias, slotLo[s], slotHi[s], ql, qh);
        for (int a = 0; a < 3; a++) { q[a][s] = ql[a]; q[3 + a][s] = qh[a]; }
    }
    memcpy(&w[0], lo, 12);
    w[3] = ebias[0] | (ebias[1] << 8) | (ebias[2] << 16) | (imask << 24);
    w[4] = childBase; w[5] = triBase;
    memcpy(&w[6], meta, 8);
    memcpy(&w[8], q[0], 8);  memcpy(&w[10], q[1], 8);     // qlo.x | qlo.y
    memcpy(&w[12], q[2], 8); memcpy(&w[14], q[3], 8);     // qlo.z | qhi.x
    memcpy(&w[16], q[4], 8); memcpy(&w[18], q[5], 8);     // qhi.y | qhi.z
}

// Binned-SAH BVH2 -> greedy 8-wide collapse -> octant slot assignment -> quantisation.  Host only.
void buildBvh8(const std::vector<BuildTriangle>& tris, Bvh8& out);

// Surface-area-heuristic expectations of a tree (MacDonald & Booth) for a random ray that hits the root box [rootLo, rootHi]: a node is visited with probability
// area(node) / area(root), using the quantised child boxes the traversal tests.  Host only; breadth-first node array (parents before children).
void bvh8SahStats(const Bvh8Node* nodes, size_t nodeCount, const float* rootLo, const float* rootHi, double* expectedNodeVisits, double* expectedTriangleTests, uint32_t* leafCount);

} // namespace pt
