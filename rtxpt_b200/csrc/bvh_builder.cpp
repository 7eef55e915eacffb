// bvh_builder.cpp — host-side acceleration-structure build, standing in for the driver-side work behind
// Sample::CreateBlases / BuildTLAS (Rtxpt/Sample.cpp:1061-1240): all instances are flattened to world space (static scenes;
// per-frame refit of animated instances is SURVEY.md §8f row 4) and one compressed 8-wide BVH is built over the triangles.
//   1. binned-SAH BVH2 (16 bins, 3 axes), leaves of at most 3 triangles, OpenMP tasks over subtrees
//   2. greedy collapse to 8 children per node (largest-area child expanded first)
//   3. children assigned to octant slots (greedy max of dot(centroid offset, slot direction))
//   4. breadth-first layout + 8-bit quantisation, conservative (floor/ceil in double)
#include "bvh8.h"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <omp.h>

namespace pt {
namespace {

struct Box
{
    float lo[3], hi[3];
    void reset() { for (int a = 0; a < 3; a++) { lo[a] = 3.0e38f; hi[a] = -3.0e38f; } }
    void grow(const float* p) { for (int a = 0; a < 3; a++) { lo[a] = std::min(lo[a], p[a]); hi[a] = std::max(hi[a], p[a]); } }
    void grow(const Box& b) { for (int a = 0; a < 3; a++) { lo[a] = std::min(lo[a], b.lo[a]); hi[a] = std::max(hi[a], b.hi[a]); } }
    float area() const { float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2]; return (dx < 0) ? 0.0f : 2.0f * (dx * dy + dy * dz + dz * dx); }
};

struct Node2 { Box box; uint32_t left, right; uint32_t first, count; };     // count > 0: leaf over order[first, first+count)

struct Builder2
{
    const std::vector<BuildTriangle>& tris;
    std::vector<Box> triBox;
    std::vector<float> cen;         // 3 per triangle
    std::vector<uint32_t> order;
    std::vector<Node2> nodes;
    std::atomic<uint32_t> nodeCount{0};

    explicit Builder2(const std::vector<BuildTriangle>& t) : tris(t) {}

    uint32_t alloc() { return nodeCount.fetch_add(1); }

    void build(uint32_t nodeIdx, uint32_t first, uint32_t count, int depth)
    {
        Node2& nd = nodes[nodeIdx];
        Box box, cbox; box.reset(); cbox.reset();
        for (uint32_t i = first; i < first + count; i++) { uint32_t id = order[i]; box.grow(triBox[id]); cbox.grow(&cen[id * 3]); }
        nd.box = box; nd.first = first; nd.count = 0; nd.left = nd.right = 0;
        if (count == 1) { nd.count = 1; return; }
        static const int NB = [] { const char* e = getenv("RTXPT_BVH_BINS"); return e ? std::min(64, std::max(4, atoi(e))) : 16; }();
        static const float travCost = [] { const char* e = getenv("RTXPT_BVH_TRAVCOST"); return e ? float(atof(e)) : 1.0f; }();
        float bestCost = 3.0e38f; int bestAxis = -1, bestSplit = -1;
        for (int axis = 0; axis < 3; axis++)
        {
            float ext = cbox.hi[axis] - cbox.lo[axis];
            if (!(ext > 0.0f)) continue;
            Box bb[64]; uint32_t bn[64];
            for (int b = 0; b < NB; b++) { bb[b].reset(); bn[b] = 0; }
            const float scale = float(NB) / ext;
            for (uint32_t i = first; i < first + count; i++)
            {
                uint32_t id = order[i];
                int b = std::min(std::max(int((cen[id * 3 + axis] - cbox.lo[axis]) * scale), 0), NB - 1);
                bb[b].grow(triBox[id]); bn[b]++;
            }
            float rightArea[64]; uint32_t rightN[64];
            Box acc; acc.reset(); uint32_t c = 0;
            for (int b = NB - 1; b > 0; b--) { acc.grow(bb[b]); c += bn[b]; rightArea[b] = acc.area(); rightN[b] = c; }
            acc.reset(); c = 0;
            for (int b = 0; b < NB - 1; b++)
            {
                acc.grow(bb[b]); c += bn[b];
                if (c == 0 || rightN[b + 1] == 0) continue;
                float cost = acc.area() * float(c) + rightArea[b + 1] * float(rightN[b + 1]);
                if (cost < bestCost) { bestCost = cost; bestAxis = axis; bestSplit = b; }
            }
        }
        if (count <= 3)
        {   // SAH termination: a leaf slot of the wide node can hold up to 3 triangles
            float leafCost = box.area() * float(count);
            float splitCost = (bestAxis >= 0) ? (bestCost + box.area() * travCost) : 3.0e38f;
            if (leafCost <= splitCost) { nd.count = count; return; }
        }
        uint32_t mid;
        if (bestAxis < 0) mid = first + count / 2;              // all centroids coincide: split arbitrarily
        else
        {
            const float lo = cbox.lo[bestAxis], scale = float(NB) / (cbox.hi[bestAxis] - cbox.lo[bestAxis]);
            const int axis = bestAxis, split = bestSplit;
            auto it = std::partition(order.begin() + first, order.begin() + first + count, [&](uint32_t id) {
                int b = std::min(std::max(int((cen[id * 3 + axis] - lo) * scale), 0), NB - 1); return b <= split; });
            mid = uint32_t(it - order.begin());
            if (mid == first || mid == first + count) mid = first + count / 2;
        }
        uint32_t l = alloc(), r = alloc();
        nodes[nodeIdx].left = l; nodes[nodeIdx].right = r;
        const uint32_t ln = mid - first, rn = first + count - mid;
        if (count > 4096 && depth < 24)
        {
            #pragma omp task shared(nodes) firstprivate(l, first, ln, depth)
            build(l, first, ln, depth + 1);
            #pragma omp task shared(nodes) firstprivate(r, mid, rn, depth)
            build(r, mid, rn, depth + 1);
            #pragma omp taskwait
        }
        else { build(l, first, ln, depth + 1); build(r, mid, rn, depth + 1); }
    }

    void run()
    {
        const uint32_t n = uint32_t(tris.size());
        triBox.resize(n); cen.resize(size_t(n) * 3); order.resize(n);
        std::iota(order.begin(), order.end(), 0u);
        #pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < int64_t(n); i++)
        {
            Box b; b.reset(); b.grow(tris[i].v0); b.grow(tris[i].v1); b.grow(tris[i].v2);
            triBox[i] = b;
            for (int a = 0; a < 3; a++) cen[i * 3 + a] = 0.5f * (b.lo[a] + b.hi[a]);
        }
        nodes.resize(size_t(n) * 2 + 1);
        uint32_t root = alloc();
        #pragma omp parallel
        {
            #pragma omp single
            build(root, 0, n, 0);
        }
    }
};

inline float biasedExpToFloat(uint32_t e) { uint32_t u = e << 23; float f; memcpy(&f, &u, 4); return f; }

} // namespace

void buildBvh8(const std::vector<BuildTriangle>& tris, Bvh8& out)
{
    auto t0 = std::chrono::steady_clock::now();
    out.nodes.clear(); out.tris.clear(); out.levelStart.clear(); out.maxDepth = 0;
    for (int a = 0; a < 3; a++) { out.sceneLo[a] = 0; out.sceneHi[a] = 0; }
    if (tris.empty())
    {
        Bvh8Node n; memset(&n, 0, sizeof(n)); out.nodes.push_back(n); out.levelStart = { 0u, 1u };
        return;
    }
    Builder2 b2(tris);
    b2.run();
    const std::vector<Node2>& N = b2.nodes;
    for (int a = 0; a < 3; a++) { out.sceneLo[a] = N[0].box.lo[a]; out.sceneHi[a] = N[0].box.hi[a]; }

    struct Pending { uint32_t node2; uint32_t depth; };
    std::vector<Pending> queue; queue.reserve(tris.size() / 2 + 16);
    queue.push_back({ 0u, 1u });
    out.nodes.reserve(tris.size() / 2 + 16);
    out.tris.reserve(tris.size());
    for (size_t qi = 0; qi < queue.size(); qi++)
    {
        const uint32_t rootIdx = queue[qi].node2; const uint32_t depth = queue[qi].depth;
        out.maxDepth = std::max(out.maxDepth, depth);
        if (out.levelStart.size() < depth) out.levelStart.push_back(uint32_t(qi));       // breadth-first: depths never decrease along the queue
        // 1. gather up to 8 children
        uint32_t child[8]; int nChild = 0;
        if (N[rootIdx].count > 0) child[nChild++] = rootIdx;       // degenerate: the whole (sub)tree is one leaf
        else { child[nChild++] = N[rootIdx].left; child[nChild++] = N[rootIdx].right; }
        while (nChild < 8)
        {
            int best = -1; float bestArea = -1.0f;
            for (int i = 0; i < nChild; i++) if (N[child[i]].count == 0) { float a = N[child[i]].box.area(); if (a > bestArea) { bestArea = a; best = i; } }
            if (best < 0) break;
            uint32_t c = child[best];
            child[best] = N[c].left; child[nChild++] = N[c].right;
        }
        // 2. octant slot assignment (bvh8.h)
        const Box& nb = N[rootIdx].box;
        float childLo[8][3], childHi[8][3];
        for (int i = 0; i < nChild; i++) for (int a = 0; a < 3; a++) { childLo[i][a] = N[child[i]].box.lo[a]; childHi[i][a] = N[child[i]].box.hi[a]; }
        int childInSlot[8]; bvh8AssignSlots(nb.lo, nb.hi, nChild, childLo, childHi, childInSlot);
        // 3. slot metadata, then the node's encoding (bvh8.h: quantisation frame and child boxes)
        Bvh8Node node;
        uint8_t meta[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }; float slotLo[8][3], slotHi[8][3];
        uint32_t imask = 0;
        const uint32_t childBase = uint32_t(queue.size());
        const uint32_t triBase = uint32_t(out.tris.size());
        uint32_t triOffset = 0;
        for (int s = 0; s < 8; s++)
        {
            int ci = childInSlot[s];
            if (ci < 0) continue;
            const Node2& c = N[child[ci]];
            for (int a = 0; a < 3; a++) { slotLo[s][a] = c.box.lo[a]; slotHi[s][a] = c.box.hi[a]; }
            if (c.count == 0)
            {
                imask |= 1u << s;
                meta[s] = uint8_t(0x38 | s);                       // 0b001_11sss: internal child, bit index 24 + slot
                queue.push_back({ child[ci], depth + 1 });
            }
            else
            {
                const uint32_t unary = (c.count == 1) ? 0x1u : (c.count == 2 ? 0x3u : 0x7u);
                meta[s] = uint8_t((unary << 5) | triOffset);
                for (uint32_t k = 0; k < c.count; k++)
                {
                    const BuildTriangle& t = tris[b2.order[c.first + k]];
                    Bvh8Tri o; memcpy(o.v0, t.v0, 12); memcpy(o.v1, t.v1, 12); memcpy(o.v2, t.v2, 12);
                    o.gid = t.gid; o.subInstanceAndFlags = t.subInstanceAndFlags; o.primitiveIndex = t.primitiveIndex;
                    out.tris.push_back(o);
                }
                triOffset += c.count;
            }
        }
        bvh8EncodeNode(nb.lo, nb.hi, slotLo, slotHi, meta, imask, childBase, triBase, node.w);
        out.nodes.push_back(node);
    }
    out.levelStart.push_back(uint32_t(out.nodes.size()));
    out.buildSeconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

void bvh8SahStats(const Bvh8Node* nodes, size_t nodeCount, const float* rootLo, const float* rootHi, double* expectedNodeVisits, double* expectedTriangleTests, uint32_t* leafCount)
{
    auto boxArea = [](const double* lo, const double* hi) { const double dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2]; return 2.0 * (dx * dy + dy * dz + dz * dx); };
    double rLo[3], rHi[3]; for (int a = 0; a < 3; a++) { rLo[a] = rootLo[a]; rHi[a] = rootHi[a]; }
    const double rootArea = std::max(boxArea(rLo, rHi), 1e-30);
    // probability of visiting node i: carried down from the parent (quantised child box area / root area); breadth-first layout = parents first
    std::vector<double> visitP(nodeCount, 0.0); if (nodeCount) visitP[0] = 1.0;
    double nodeVisits = 0, triTests = 0, leaves = 0;
    for (size_t ni = 0; ni < nodeCount; ni++)
    {
        const Bvh8Node& n = nodes[ni];
        nodeVisits += visitP[ni];
        float p[3]; memcpy(p, &n.w[0], 12);
        const uint32_t e[3] = { n.w[3] & 0xFF, (n.w[3] >> 8) & 0xFF, (n.w[3] >> 16) & 0xFF }, imask = n.w[3] >> 24, childBase = n.w[4];
        const uint8_t* meta = reinterpret_cast<const uint8_t*>(&n.w[6]); const uint8_t* q = reinterpret_cast<const uint8_t*>(&n.w[8]);
        for (int s = 0; s < 8; s++)
        {
            if (meta[s] == 0) continue;
            double lo[3], hi[3];
            for (int a = 0; a < 3; a++) { const double sc = std::ldexp(1.0, int(e[a]) - 127); lo[a] = p[a] + q[a * 8 + s] * sc; hi[a] = p[a] + q[(3 + a) * 8 + s] * sc; }
            const double pr = std::min(1.0, boxArea(lo, hi) / rootArea);
            if (imask & (1u << s)) visitP[childBase + __builtin_popcount(imask & ((1u << s) - 1u))] = pr;
            else { const int cnt = __builtin_popcount(uint32_t(meta[s] >> 5)); triTests += pr * cnt; leaves += 1; }
        }
    }
    *expectedNodeVisits = nodeVisits; *expectedTriangleTests = triTests; *leafCount = uint32_t(leaves);
}

} // namespace pt

// ---- inspection hook (host only): surface-area-heuristic statistics of the tree built over a triangle soup (bvh8SahStats) -----------------------------------------------
#include "../../include/rtxpt_b200.h"
extern "C" RTXPT_API int rtxpt_b200_debug_bvh_stats(const float* triangleVertices, uint32_t triangleCount, RtxptBvhStats* out)
{
    if ((!triangleVertices && triangleCount) || !out) return RTXPT_ERR_INVALID_ARGUMENT;
    using namespace pt;
    std::vector<BuildTriangle> tris(triangleCount);
    for (uint32_t i = 0; i < triangleCount; i++)
    {
        memcpy(tris[i].v0, triangleVertices + size_t(i) * 9, 12); memcpy(tris[i].v1, triangleVertices + size_t(i) * 9 + 3, 12); memcpy(tris[i].v2, triangleVertices + size_t(i) * 9 + 6, 12);
        tris[i].gid = i; tris[i].subInstanceAndFlags = 0; tris[i].primitiveIndex = i;
    }
    Bvh8 bvh; buildBvh8(tris, bvh);
    memset(out, 0, sizeof(*out));
    out->nodeCount = uint32_t(bvh.nodes.size()); out->triangleReferenceCount = uint32_t(bvh.tris.size()); out->buildSeconds = float(bvh.buildSeconds); out->maxDepth = bvh.maxDepth;
    if (triangleCount == 0) return RTXPT_OK;
    double nodeVisits = 0, triTests = 0;
    bvh8SahStats(bvh.nodes.data(), bvh.nodes.size(), bvh.sceneLo, bvh.sceneHi, &nodeVisits, &triTests, &out->leafCount);
    out->expectedNodeVisits = float(nodeVisits); out->expectedTriangleTests = float(triTests);
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_debug_build_bvh(const float* triangleVertices, uint32_t triangleCount, void* outNodes, void* outTris, uint32_t* outLevelStart, uint32_t* outNodeCount, uint32_t* outTriCount,
                                                    uint32_t* outLevelCount)
{
    if ((!triangleVertices && triangleCount) || !outNodeCount || !outTriCount || !outLevelCount) return RTXPT_ERR_INVALID_ARGUMENT;
    using namespace pt;
    std::vector<BuildTriangle> tris(triangleCount);
    for (uint32_t i = 0; i < triangleCount; i++)
    {
        memcpy(tris[i].v0, triangleVertices + size_t(i) * 9, 12); memcpy(tris[i].v1, triangleVertices + size_t(i) * 9 + 3, 12); memcpy(tris[i].v2, triangleVertices + size_t(i) * 9 + 6, 12);
        tris[i].gid = i; tris[i].subInstanceAndFlags = 0; tris[i].primitiveIndex = i;
    }
    Bvh8 bvh; buildBvh8(tris, bvh);
    *outNodeCount = uint32_t(bvh.nodes.size()); *outTriCount = uint32_t(bvh.tris.size()); *outLevelCount = uint32_t(bvh.levelStart.size()) - 1;
    if (outNodes) memcpy(outNodes, bvh.nodes.data(), bvh.nodes.size() * sizeof(Bvh8Node));
    if (outTris) memcpy(outTris, bvh.tris.data(), bvh.tris.size() * sizeof(Bvh8Tri));
    if (outLevelStart) memcpy(outLevelStart, bvh.levelStart.data(), bvh.levelStart.size() * 4);
    return RTXPT_OK;
}
