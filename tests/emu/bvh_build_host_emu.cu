// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of the product's BVH rebuild bodies (rtxpt_b200/csrc/bvh_build.cuh: __host__ __device__ functions, the same source the CUDA kernels wrap) in the order of
// launchBvhBuild (bvh_build_kernels.cu), element by element on the CPU, plus the product's SAH statistics (bvh_builder.cpp: bvh8SahStats).  tests/test_bvh_rebuild.py holds the
// rebuild to the tree contract with it without a GPU; tests/test_gpu_bvh_rebuild.py holds the device build to it word for word.  Built by bvh_build.mk.
#include "../../rtxpt_b200/csrc/bvh_build.cuh"
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

// The radix sort is a stable counting sort per digit (a stable sort has one result, however it is computed), the exclusive scans are serial.  srcTris: n leaf triangles of 12 words in
// any order; outputs sized for n nodes / triangles and 33 level starts.  Returns 0, 1 (deeper than bvhb::kMaxDepth levels: not built) or 2 (the clustering stalled).
extern "C" int emu_build_bvh(const float* srcTris, uint32_t n, uint32_t* outNodes, float* outTris, float* outNodeBox, uint32_t* outLevelStart, uint32_t* outNodeCount, uint32_t* outLevelCount,
                             uint32_t* outIterations)
{
    using namespace pt::bvhb;
    if (n == 0) return -1;
    std::vector<float4> tris(size_t(n) * 3), outT(size_t(n) * 3); std::vector<uint4> nodes(size_t(n) * 5); std::vector<float> nodeBox(size_t(n) * 6), box2(size_t(n) * 12);
    std::vector<u64> keys[2] = { std::vector<u64>(n), std::vector<u64>(n) }, flags(n), misc(2);
    std::vector<uint32_t> vals[2] = { std::vector<uint32_t>(n), std::vector<uint32_t>(n) }, clusters[2] = { std::vector<uint32_t>(n), std::vector<uint32_t>(n) };
    std::vector<uint32_t> count2(size_t(n) * 2), nn(n), nodeRoot(n), cen(6); std::vector<uint2> child2(n);
    Params p{};
    p.srcTris = reinterpret_cast<const float4*>(srcTris); p.tris = tris.data(); p.triCount = n; p.cenBounds = cen.data(); p.varying = misc.data() + 1;
    for (int k = 0; k < 2; k++) { p.keys[k] = keys[k].data(); p.vals[k] = vals[k].data(); p.clusters[k] = clusters[k].data(); }
    p.box2 = box2.data(); p.child2 = child2.data(); p.count2 = count2.data(); p.nn = nn.data(); p.flags = flags.data(); p.nodeRoot = nodeRoot.data(); p.levelCounts = flags.data();
    p.nodes = nodes.data(); p.outTris = outT.data(); p.nodeBox = nodeBox.data();
    auto scan = [](u64* a, uint32_t m) { u64 t = 0; for (uint32_t i = 0; i < m; i++) { const u64 v = a[i]; a[i] = t; t += v; } return t; };
    for (uint32_t i = 0; i < n; i++) scatterByGid(p, i);
    for (int a = 0; a < 3; a++) { cen[a] = 0xFFFFFFFFu; cen[3 + a] = 0; }
    for (uint32_t g = 0; g < n; g++) { uint32_t k[3]; centroidKeys(p, g, k); for (int a = 0; a < 3; a++) { cen[a] = std::min(cen[a], k[a]); cen[3 + a] = std::max(cen[3 + a], k[a]); } }
    const u64 key0 = mortonCode(p, 0); u64 varying = 0;
    for (uint32_t g = 0; g < n; g++) { keys[0][g] = mortonCode(p, g); vals[0][g] = g; varying |= keys[0][g] ^ key0; }
    int cur = 0;
    for (uint32_t shift = 0; shift < 64; shift += 8)
    {
        if (((varying >> shift) & 0xFFu) == 0) continue;
        uint32_t off[257] = {};
        for (uint32_t i = 0; i < n; i++) off[radixDigit(keys[cur][i], shift) + 1]++;
        for (int d = 0; d < 256; d++) off[d + 1] += off[d];
        for (uint32_t i = 0; i < n; i++) { const uint32_t dst = off[radixDigit(keys[cur][i], shift)]++; keys[cur ^ 1][dst] = keys[cur][i]; vals[cur ^ 1][dst] = vals[cur][i]; }
        cur ^= 1;
    }
    p.sorted = vals[cur].data();
    for (uint32_t k = 0; k < n; k++) leafInit(p, k);
    uint32_t count = n, nextNode = n, iterations = 0; int src = 0;
    while (count > 1)
    {
        #pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < int64_t(count); i++) nearestNeighbour(p, clusters[src].data(), count, uint32_t(i));
        for (uint32_t i = 0; i < count; i++) mergeFlags(p, i);
        const u64 total = scan(flags.data(), count);
        #pragma omp parallel for schedule(static)
        for (int64_t i = 0; i < int64_t(count); i++) mergeStep(p, clusters[src].data(), clusters[src ^ 1].data(), uint32_t(i), nextNode);
        const uint32_t merges = uint32_t(total >> 32);
        if (merges == 0) return 2;
        nextNode += merges; count = uint32_t(total); src ^= 1; iterations++;
    }
    nodeRoot[0] = n > 1 ? 2 * n - 2 : 0u;
    std::vector<uint32_t> levelStart = { 0u };
    uint32_t first = 0, end = 1, triRunning = 0;
    for (;;)
    {
        if (levelStart.size() > kMaxDepth) return 1;
        for (uint32_t ni = first; ni < end; ni++) collapseCount(p, ni, first);
        const u64 total = scan(flags.data(), end - first);
        for (uint32_t ni = first; ni < end; ni++) collapseEmit(p, ni, first, end, triRunning);
        levelStart.push_back(end);
        const uint32_t next = uint32_t(total >> 32); triRunning += uint32_t(total);
        if (next == 0) break;
        first = end; end += next;
    }
    if (triRunning != n) return 2;
    for (size_t d = levelStart.size() - 1; d-- > 0;) for (uint32_t ni = levelStart[d]; ni < levelStart[d + 1]; ni++) encodeNode(p, ni);
    memcpy(outNodes, nodes.data(), size_t(end) * 80); memcpy(outTris, outT.data(), size_t(n) * 48); memcpy(outNodeBox, nodeBox.data(), size_t(end) * 24);
    memcpy(outLevelStart, levelStart.data(), levelStart.size() * 4);
    *outNodeCount = end; *outLevelCount = uint32_t(levelStart.size()) - 1; *outIterations = iterations;
    return 0;
}

// the product's SAH statistics (bvh_builder.cpp: bvh8SahStats) of a node array over a root box
extern "C" int emu_bvh_stats(const uint32_t* nodes, uint32_t nodeCount, const float* rootBox, double* outVisitsTests, uint32_t* outLeafCount)
{
    pt::bvh8SahStats(reinterpret_cast<const pt::Bvh8Node*>(nodes), nodeCount, rootBox, rootBox + 3, &outVisitsTests[0], &outVisitsTests[1], outLeafCount);
    return 0;
}
