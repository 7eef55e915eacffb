// bvh_build.cuh - device rebuild of the compressed 8-wide BVH over the context's current leaf triangles (rtxpt_b200_rebuild_bvh), producing the tree format of bvh8.h that the
// traversal, the refit and the shared-memory staging read.  Bodies are __host__ __device__ over one parameter block (kernels and launch sequence: bvh_build_kernels.cu; host
// build: tests/emu), every one a function of its own element, so the host build and the device give the same words.
//   1. the leaf triangles scattered to their gid position (gids are a dense permutation), centroid bounds (exact min / max), 63-bit Morton codes (21 bits per axis)
//   2. stable LSD radix sort of (Morton code, gid), 8 bits per pass: equal codes stay in gid order
//   3. PLOC (Meister & Bittner, "Parallel Locally-Ordered Clustering for Bounding Volume Hierarchy Construction", TVCG 2018): every cluster finds the neighbour within
//      +-kPlocRadius positions whose merged box has the smallest surface area (ties: nearestNeighbour); mutual pairs merge, survivors are compacted by a scan.  A merge
//      of at most 3 triangles becomes one leaf under the host builder's SAH rule (bvh_builder.cpp)
//   4. top-down collapse, one breadth-first level per launch: the host builder's greedy expansion, slot assignment (bvh8AssignSlots), childBase / triBase from scans
//   5. bottom-up encoding, deepest level first: exact child boxes from the leaf triangles (as refit.cuh computes them) and bvh8EncodeNode, so an identity refit returns the tree
// No float atomics, no atomic counters: the tree is a function of the triangles alone, whatever their current leaf order.
#pragma once
#include "device_math.cuh"
#include "bvh8.h"
#include <string.h>
#include <vector>

namespace pt { namespace bvhb {

typedef unsigned long long u64;
constexpr uint kLeafFlag = 0x80000000u;         // count2: the subtree is one leaf of (count & ~kLeafFlag) triangles
constexpr uint kPlocRadius = 16;
constexpr uint kMaxDepth = 32;                  // traverse.cuh: kTraversalStackSize; a deeper tree could overflow the traversal stack
constexpr uint kRadixTile = 256;

struct Params
{
    const float4* srcTris;          // current leaf triangles, leaf order: 3 float4 each, gid in .w of the first
    float4* tris;                   // the same records in gid order
    uint triCount;
    uint* cenBounds;                // 6 ordered keys (orderedKey): centroid min xyz, max xyz
    u64* varying;                   // OR over all triangles of (Morton code ^ Morton code of gid 0)
    u64* keys[2]; uint* vals[2];    // radix sort ping-pong: Morton code, gid
    u64* hist;                      // digit counts of one pass, digit-major: [256][tiles]
    const uint* sorted;             // gids in Morton order (the sort's output)
    float* box2; uint2* child2; uint* count2;   // BVH2: leaves 0..n-1 (sorted position), internal nodes n..2n-2; child2 indexed by node - n; count2: triangles | kLeafFlag
    uint* clusters[2]; uint* nn; u64* flags;    // PLOC: cluster nodes by position, nearest neighbour, (merge << 32 | keep) then their exclusive scan
    uint* nodeRoot;                 // BVH2 node of each BVH8 node
    u64* levelCounts;               // per node of the level being collapsed: (internal children << 32 | leaf triangles), then their exclusive scan
    uint4* nodes; float4* outTris; float* nodeBox;      // the new tree: nodes, leaf triangles, exact node boxes (6 floats per node)
};

#ifdef __CUDA_ARCH__
PT_HD uint asUint(float f) { return __float_as_uint(f); }
PT_HD float asFloat(uint u) { return __uint_as_float(u); }
PT_HD uint popc(uint v) { return uint(__popc(v)); }
#else
PT_HD uint asUint(float f) { uint u; memcpy(&u, &f, 4); return u; }
PT_HD float asFloat(uint u) { float f; memcpy(&f, &u, 4); return f; }
PT_HD uint popc(uint v) { return uint(__builtin_popcount(v)); }
#endif
// float <-> unsigned key with the same order (-0 below +0): exact min / max reductions by integer comparison
PT_HD uint orderedKey(float f) { const uint u = asUint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
PT_HD float orderedFloat(uint k) { return asFloat((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }
PT_HD float minf(float a, float b) { return b < a ? b : a; }      // std::min / std::max, as the host builder's boxes
PT_HD float maxf(float a, float b) { return a < b ? b : a; }
PT_HD float comp(const float4& v, int a) { return a == 0 ? v.x : (a == 1 ? v.y : v.z); }

PT_HD void triangleBox(const float4* t, float* lo, float* hi)
{
    for (int a = 0; a < 3; a++) { lo[a] = 3.0e38f; hi[a] = -3.0e38f; }
    for (int k = 0; k < 3; k++) for (int a = 0; a < 3; a++) { lo[a] = minf(lo[a], comp(t[k], a)); hi[a] = maxf(hi[a], comp(t[k], a)); }
}
// surface area of a box, as the host builder's Box::area
PT_HD float boxArea(const float* lo, const float* hi)
{
    const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
    return (dx < 0) ? 0.0f : 2.0f * (dx * dy + dy * dz + dz * dx);
}

// ---- 1. gid order, centroid bounds, Morton codes -------------------------------------------------------------------------------------------------------------------------------
PT_HD void scatterByGid(const Params& p, uint i)
{
    const uint g = asUint(p.srcTris[size_t(i) * 3].w);
    for (int k = 0; k < 3; k++) p.tris[size_t(g) * 3 + k] = p.srcTris[size_t(i) * 3 + k];
}
// centroid (box centre, as the host builder) of triangle g, as ordered keys
PT_HD void centroidKeys(const Params& p, uint g, uint* key)
{
    float lo[3], hi[3]; triangleBox(p.tris + size_t(g) * 3, lo, hi);
    for (int a = 0; a < 3; a++) key[a] = orderedKey(0.5f * (lo[a] + hi[a]));
}
PT_HD u64 spreadBits21(u64 v)
{
    v &= 0x1FFFFFull;
    v = (v | (v << 32)) & 0x1F00000000FFFFull;
    v = (v | (v << 16)) & 0x1F0000FF0000FFull;
    v = (v | (v << 8)) & 0x100F00F00F00F00Full;
    v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
    v = (v | (v << 2)) & 0x1249249249249249ull;
    return v;
}
// 63-bit Morton code of triangle g's centroid in the centroid bounds (cenBounds after the reduction); exact double arithmetic on both sides
PT_HD u64 mortonCode(const Params& p, uint g)
{
    uint key[3]; centroidKeys(p, g, key);
    u64 q[3];
    for (int a = 0; a < 3; a++)
    {
        const double lo = double(orderedFloat(p.cenBounds[a])), ext = double(orderedFloat(p.cenBounds[3 + a])) - lo;
        const double t = ext > 0.0 ? (double(orderedFloat(key[a])) - lo) / ext * 2097152.0 : 0.0;
        q[a] = u64(t < 2097151.0 ? (t > 0.0 ? t : 0.0) : 2097151.0);
    }
    return (spreadBits21(q[0]) << 2) | (spreadBits21(q[1]) << 1) | spreadBits21(q[2]);
}
PT_HD uint radixDigit(u64 key, uint shift) { return uint(key >> shift) & 0xFFu; }

// ---- 3. PLOC ----------------------------------------------------------------------------------------------------------------------------------------------------------------------
// BVH2 leaf k: the k-th triangle in Morton order; every leaf starts as its own cluster
PT_HD void leafInit(const Params& p, uint k)
{
    float lo[3], hi[3]; triangleBox(p.tris + size_t(p.sorted[k]) * 3, lo, hi);
    for (int a = 0; a < 3; a++) { p.box2[size_t(k) * 6 + a] = lo[a]; p.box2[size_t(k) * 6 + 3 + a] = hi[a]; }
    p.count2[k] = 1u | kLeafFlag; p.clusters[0][k] = k;
}
PT_HD float mergedArea(const Params& p, uint a, uint b)
{
    const float* A = p.box2 + size_t(a) * 6; const float* B = p.box2 + size_t(b) * 6;
    float lo[3], hi[3]; for (int k = 0; k < 3; k++) { lo[k] = minf(A[k], B[k]); hi[k] = maxf(A[3 + k], B[3 + k]); }
    return boxArea(lo, hi);
}
// position of cluster i's nearest neighbour among positions i - r .. i + r of n: the smallest merged area; on equal areas the nearer position, then the pair that starts at an
// even position, then the smaller position.  (area, distance, parity, position) orders the pairs strictly, so the smallest pair is mutual and every iteration merges; and a run of
// equal boxes (an instance scaled to a point, identical triangles) pairs off (2k, 2k + 1) and halves, where "smaller position first" alone would merge one pair per iteration and
// build a chain one level deeper per triangle.
PT_HD void nearestNeighbour(const Params& p, const uint* cl, uint n, uint i)
{
    const uint lo = i > kPlocRadius ? i - kPlocRadius : 0u, hi = (i + kPlocRadius < n) ? i + kPlocRadius : n - 1;
    const uint ci = cl[i];
    float best = 0.0f; uint bj = 0, bd = 0, bm = 0;
    bool first = true;
    for (uint j = lo; j <= hi; j++)
    {
        if (j == i) continue;
        const float a = mergedArea(p, ci, cl[j]);
        const uint d = j < i ? i - j : j - i, m = j < i ? j : i;
        const bool better = first || a < best || (a == best && (d < bd || (d == bd && ((m & 1u) < (bm & 1u) || ((m & 1u) == (bm & 1u) && m < bm)))));
        if (better) { best = a; bj = j; bd = d; bm = m; first = false; }
    }
    p.nn[i] = bj;
}
PT_HD void mergeFlags(const Params& p, uint i)
{
    const uint j = p.nn[i]; const bool mutual = p.nn[j] == i;
    p.flags[i] = (u64(mutual && i < j) << 32) | u64(!(mutual && i > j));
}
// BVH2 node `id` over clusters l and r; a subtree of at most 3 triangles becomes one leaf when area * n <= area * 1 + area_l * n_l + area_r * n_r (bvh_builder.cpp)
PT_HD void makeNode(const Params& p, uint id, uint l, uint r)
{
    const float* L = p.box2 + size_t(l) * 6; const float* R = p.box2 + size_t(r) * 6; float* B = p.box2 + size_t(id) * 6;
    float lo[3], hi[3]; for (int k = 0; k < 3; k++) { lo[k] = minf(L[k], R[k]); hi[k] = maxf(L[3 + k], R[3 + k]); }
    for (int k = 0; k < 3; k++) { B[k] = lo[k]; B[3 + k] = hi[k]; }
    const uint nl = p.count2[l] & ~kLeafFlag, nr = p.count2[r] & ~kLeafFlag, n = nl + nr;
    const float area = boxArea(lo, hi);
    const bool leaf = n <= 3 && area * float(n) <= (boxArea(L, L + 3) * float(nl) + boxArea(R, R + 3) * float(nr)) + area * 1.0f;
    p.count2[id] = n | (leaf ? kLeafFlag : 0u);
    p.child2[id - p.triCount] = make_uint2(l, r);
}
// after the scan of flags: mutual pairs (lower position) make node nextNode + merge offset; kept clusters move to their compacted position in dst
PT_HD void mergeStep(const Params& p, const uint* src, uint* dst, uint i, uint nextNode)
{
    const uint j = p.nn[i]; const bool mutual = p.nn[j] == i;
    const u64 off = p.flags[i];
    uint id = src[i];
    if (mutual && i < j) { id = nextNode + uint(off >> 32); makeNode(p, id, src[i], src[j]); }
    if (!(mutual && i > j)) dst[uint(off)] = id;
}

// ---- 4. top-down collapse --------------------------------------------------------------------------------------------------------------------------------------------------------
PT_HD bool isLeaf(const Params& p, uint node) { return (p.count2[node] & kLeafFlag) != 0; }
// up to 8 children of BVH2 node `root`: the host builder's greedy rule (expand the internal child of largest area, first on ties); childInSlot: bvh8AssignSlots
PT_HD int gatherChildren(const Params& p, uint root, uint* child, int* childInSlot)
{
    int nChild = 0;
    if (isLeaf(p, root)) child[nChild++] = root;                // the whole tree is one leaf
    else { const uint2 c = p.child2[root - p.triCount]; child[nChild++] = c.x; child[nChild++] = c.y; }
    while (nChild < 8)
    {
        int best = -1; float bestArea = -1.0f;
        for (int i = 0; i < nChild; i++) if (!isLeaf(p, child[i])) { const float* b = p.box2 + size_t(child[i]) * 6; const float a = boxArea(b, b + 3); if (a > bestArea) { bestArea = a; best = i; } }
        if (best < 0) break;
        const uint2 c = p.child2[child[best] - p.triCount];
        child[best] = c.x; child[nChild++] = c.y;
    }
    float clo[8][3], chi[8][3];
    for (int i = 0; i < nChild; i++) for (int a = 0; a < 3; a++) { clo[i][a] = p.box2[size_t(child[i]) * 6 + a]; chi[i][a] = p.box2[size_t(child[i]) * 6 + 3 + a]; }
    const float* rb = p.box2 + size_t(root) * 6;
    bvh8AssignSlots(rb, rb + 3, nChild, clo, chi, childInSlot);
    return nChild;
}
// pass 1 of a level: what node ni needs of the level's scans
PT_HD void collapseCount(const Params& p, uint ni, uint first)
{
    uint child[8]; int childInSlot[8];
    const int nChild = gatherChildren(p, p.nodeRoot[ni], child, childInSlot);
    uint internal = 0, tris = 0;
    for (int i = 0; i < nChild; i++) { if (isLeaf(p, child[i])) tris += p.count2[child[i]] & ~kLeafFlag; else internal++; }
    p.levelCounts[ni - first] = (u64(internal) << 32) | tris;
}
// triangles of a leaf subtree (at most 3), left first, as sorted positions
PT_HD uint leafTriangles(const Params& p, uint node, uint* out)
{
    uint stack[4]; int sp = 0; uint m = 0;
    stack[sp++] = node;
    while (sp > 0)
    {
        const uint c = stack[--sp];
        if (c < p.triCount) { out[m++] = c; continue; }
        const uint2 ch = p.child2[c - p.triCount]; stack[sp++] = ch.y; stack[sp++] = ch.x;
    }
    return m;
}
// pass 2 of a level, after the scans: childBase / triBase, slot metadata, the next level's BVH2 roots, the leaf triangles copied whole into leaf order
PT_HD void collapseEmit(const Params& p, uint ni, uint first, uint end, uint triRunning)
{
    uint child[8]; int childInSlot[8];
    gatherChildren(p, p.nodeRoot[ni], child, childInSlot);
    const u64 off = p.levelCounts[ni - first];
    const uint childBase = end + uint(off >> 32), triBase = triRunning + uint(off);
    uint meta[2] = { 0, 0 }, imask = 0, k = 0, triOffset = 0;
    for (int s = 0; s < 8; s++)
    {
        if (childInSlot[s] < 0) continue;
        const uint c = child[childInSlot[s]];
        uint m;
        if (!isLeaf(p, c)) { imask |= 1u << s; m = 0x38u | uint(s); p.nodeRoot[childBase + k++] = c; }
        else
        {
            uint pos[3]; const uint cnt = leafTriangles(p, c, pos);
            m = (((cnt == 1) ? 0x1u : (cnt == 2 ? 0x3u : 0x7u)) << 5) | triOffset;
            for (uint t = 0; t < cnt; t++) for (int q = 0; q < 3; q++) p.outTris[size_t(triBase + triOffset + t) * 3 + q] = p.tris[size_t(p.sorted[pos[t]]) * 3 + q];
            triOffset += cnt;
        }
        meta[s >> 2] |= m << ((s & 3) * 8);
    }
    uint4* n = p.nodes + size_t(ni) * 5;
    n[0] = make_uint4(0, 0, 0, imask << 24);
    n[1] = make_uint4(childBase, triBase, meta[0], meta[1]);
}

// ---- 5. bottom-up encoding: the exact box of every child (leaf: its triangles' vertices; internal: the child's box, encoded before), as refit.cuh's refitNode computes them ----------
PT_HD void encodeNode(const Params& p, uint ni)
{
    uint4* n = p.nodes + size_t(ni) * 5;
    const uint4 n0 = n[0], n1 = n[1];
    const uint imask = n0.w >> 24, childBase = n1.x, triBase = n1.y;
    uint8_t meta[8];
    float clo[8][3], chi[8][3];
    float lo[3] = { 3.0e38f, 3.0e38f, 3.0e38f }, hi[3] = { -3.0e38f, -3.0e38f, -3.0e38f };
    for (int s = 0; s < 8; s++)
    {
        meta[s] = uint8_t(((s < 4 ? n1.z : n1.w) >> ((s & 3) * 8)) & 0xFFu);
        if (meta[s] == 0) continue;
        for (int a = 0; a < 3; a++) { clo[s][a] = 3.0e38f; chi[s][a] = -3.0e38f; }
        if (imask & (1u << s))
        {
            const float* b = p.nodeBox + size_t(childBase + popc(imask & ((1u << s) - 1u))) * 6;
            for (int a = 0; a < 3; a++) { clo[s][a] = b[a]; chi[s][a] = b[3 + a]; }
        }
        else
        {
            const uint first = triBase + (meta[s] & 31u), count = popc(uint(meta[s]) >> 5);
            for (uint t = first; t < first + count; t++) for (int k = 0; k < 3; k++)
            {
                const float4 v = p.outTris[size_t(t) * 3 + k]; const float c[3] = { v.x, v.y, v.z };
                for (int a = 0; a < 3; a++) { clo[s][a] = fminf(clo[s][a], c[a]); chi[s][a] = fmaxf(chi[s][a], c[a]); }
            }
        }
        for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], clo[s][a]); hi[a] = fmaxf(hi[a], chi[s][a]); }
    }
    float* box = p.nodeBox + size_t(ni) * 6;
    for (int a = 0; a < 3; a++) { box[a] = lo[a]; box[3 + a] = hi[a]; }
    uint w[20];
    bvh8EncodeNode(lo, hi, clo, chi, meta, imask, childBase, triBase, w);
    for (int k = 0; k < 5; k++) n[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
}

} // namespace bvhb

// launch sequence (bvh_build_kernels.cu): scanBlocks holds ceil(max(n, 256 * ceil(n / 256)) / kScanBlock) entries, misc 1
struct BvhBuildScans { bvhb::u64* scanBlocks; bvhb::u64* misc; };
struct BvhBuildResult
{
    enum { kOk = 0, kTooDeep = 1, kStalled = 2 };
    int status = kOk;
    uint32_t nodeCount = 0, rootNode2 = 0, plocIterations = 0, radixPasses = 0, syncs = 0;
    std::vector<uint32_t> levelStart;
    float rootBox[6] = {};          // exact box of the root (sceneDiagonal, the SAH statistics)
};
cudaError_t launchBvhBuild(bvhb::Params p, const BvhBuildScans& scans, int smCount, cudaStream_t s, BvhBuildResult& r);

} // namespace pt
