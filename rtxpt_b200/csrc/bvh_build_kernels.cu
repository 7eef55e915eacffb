// bvh_build_kernels.cu - device rebuild of the CWBVH8 (bodies: bvh_build.cuh).  Grid-stride kernels over triangles, clusters or the nodes of one level; the radix sort works on
// tiles of 256 keys (stable ranks from warp matches); every compaction and allocation is an exclusive scan (scan.cuh).  The host reads a count back after every PLOC iteration and
// every tree level (8 to 16 bytes each) to size the next launches.  Compiled once with IEEE arithmetic (-fmad=false) and linked into both libraries, like the refit, so that the
// device tree equals the host build of the same bodies word for word.
#include "bvh_build.cuh"
#include "scan.cuh"
#include <algorithm>

namespace pt { namespace bvhb {

static unsigned gridFor(uint n, int smCount) { return std::max(1u, std::min((n + 255) / 256, unsigned(smCount) * 8)); }

__global__ void __launch_bounds__(256) k_bvhb_scatter(const __grid_constant__ Params p)
{
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < p.triCount; i += gridDim.x * 256) scatterByGid(p, i);
}
__global__ void __launch_bounds__(256) k_bvhb_bounds(const __grid_constant__ Params p)
{
    uint mn[3] = { 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu }, mx[3] = { 0, 0, 0 };
    for (uint g = blockIdx.x * 256 + threadIdx.x; g < p.triCount; g += gridDim.x * 256)
    {
        uint k[3]; centroidKeys(p, g, k);
        for (int a = 0; a < 3; a++) { mn[a] = min(mn[a], k[a]); mx[a] = max(mx[a], k[a]); }
    }
    for (int a = 0; a < 3; a++) { mn[a] = __reduce_min_sync(0xFFFFFFFFu, mn[a]); mx[a] = __reduce_max_sync(0xFFFFFFFFu, mx[a]); }
    if ((threadIdx.x & 31) == 0) for (int a = 0; a < 3; a++) { atomicMin(p.cenBounds + a, mn[a]); atomicMax(p.cenBounds + 3 + a, mx[a]); }      // integer min / max: order-free
}
__global__ void __launch_bounds__(256) k_bvhb_morton(const __grid_constant__ Params p)
{
    const u64 key0 = mortonCode(p, 0);
    u64 diff = 0;
    for (uint g = blockIdx.x * 256 + threadIdx.x; g < p.triCount; g += gridDim.x * 256)
    {
        const u64 key = mortonCode(p, g);
        p.keys[0][g] = key; p.vals[0][g] = g; diff |= key ^ key0;
    }
    const uint lo = __reduce_or_sync(0xFFFFFFFFu, uint(diff)), hi = __reduce_or_sync(0xFFFFFFFFu, uint(diff >> 32));
    if ((threadIdx.x & 31) == 0 && (lo | hi)) atomicOr(p.varying, (u64(hi) << 32) | lo);
}
// one tile of 256 keys per CTA: per-warp digit counts (warp match), the tile's histogram and each key's stable rank within the tile
__device__ __forceinline__ uint tileRank(const u64* keys, uint n, uint shift, uint (*cnt)[256], uint& digit, bool& inside)
{
    const uint i = blockIdx.x * kRadixTile + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int w = 0; w < 8; w++) cnt[w][threadIdx.x] = 0;
    __syncthreads();
    inside = i < n; digit = inside ? radixDigit(keys[i], shift) : 0x100u;
    const uint peers = __match_any_sync(0xFFFFFFFFu, digit);
    if (inside && lane == uint(__ffs(peers) - 1)) cnt[warp][digit] = uint(__popc(peers));
    __syncthreads();
    uint rank = uint(__popc(peers & ((1u << lane) - 1u)));
    if (inside) for (uint w = 0; w < warp; w++) rank += cnt[w][digit];
    return rank;
}
__global__ void __launch_bounds__(256) k_bvhb_radix_hist(const u64* keys, uint n, uint shift, u64* hist, uint tiles)
{
    __shared__ uint cnt[8][256];
    uint digit; bool inside; tileRank(keys, n, shift, cnt, digit, inside);
    uint total = 0; for (int w = 0; w < 8; w++) total += cnt[w][threadIdx.x];
    hist[size_t(threadIdx.x) * tiles + blockIdx.x] = total;
}
__global__ void __launch_bounds__(256) k_bvhb_radix_scatter(const u64* keys, const uint* vals, u64* keysOut, uint* valsOut, uint n, uint shift, const u64* hist, uint tiles)
{
    __shared__ uint cnt[8][256];
    uint digit; bool inside; const uint rank = tileRank(keys, n, shift, cnt, digit, inside);
    if (!inside) return;
    const uint i = blockIdx.x * kRadixTile + threadIdx.x, dst = uint(hist[size_t(digit) * tiles + blockIdx.x]) + rank;
    keysOut[dst] = keys[i]; valsOut[dst] = vals[i];
}
__global__ void __launch_bounds__(256) k_bvhb_leaves(const __grid_constant__ Params p)
{
    for (uint k = blockIdx.x * 256 + threadIdx.x; k < p.triCount; k += gridDim.x * 256) leafInit(p, k);
}
__global__ void __launch_bounds__(256) k_bvhb_ploc_nn(const __grid_constant__ Params p, const uint* cl, uint n)
{
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) nearestNeighbour(p, cl, n, i);
}
__global__ void __launch_bounds__(256) k_bvhb_ploc_flags(const __grid_constant__ Params p, uint n)
{
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) mergeFlags(p, i);
}
__global__ void __launch_bounds__(256) k_bvhb_ploc_merge(const __grid_constant__ Params p, const uint* src, uint* dst, uint n, uint nextNode)
{
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) mergeStep(p, src, dst, i, nextNode);
}
__global__ void __launch_bounds__(128) k_bvhb_collapse_count(const __grid_constant__ Params p, uint first, uint end)
{
    for (uint ni = first + blockIdx.x * 128 + threadIdx.x; ni < end; ni += gridDim.x * 128) collapseCount(p, ni, first);
}
__global__ void __launch_bounds__(128) k_bvhb_collapse_emit(const __grid_constant__ Params p, uint first, uint end, uint triRunning)
{
    for (uint ni = first + blockIdx.x * 128 + threadIdx.x; ni < end; ni += gridDim.x * 128) collapseEmit(p, ni, first, end, triRunning);
}
__global__ void __launch_bounds__(128) k_bvhb_encode(const __grid_constant__ Params p, uint first, uint end)
{
    for (uint ni = first + blockIdx.x * 128 + threadIdx.x; ni < end; ni += gridDim.x * 128) encodeNode(p, ni);
}

} // namespace bvhb

// the whole build on stream s; returns after the stream has drained.  scanBlocks: ceil(max(256 * tiles, n) / kScanBlock) entries; misc: 2 entries
cudaError_t launchBvhBuild(bvhb::Params p, const BvhBuildScans& scratch, int smCount, cudaStream_t s, BvhBuildResult& r)
{
    using namespace bvhb;
    const uint n = p.triCount;
    r = BvhBuildResult{};
    u64 host[2] = { 0, 0 };
    auto readback = [&](const u64* src, int count) -> cudaError_t {
        cudaError_t e = cudaMemcpyAsync(host, src, size_t(count) * 8, cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        r.syncs++;
        return e;
    };
#define BVHB_CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return e_; } while (0)
    // 1. gid order, centroid bounds, Morton codes and the bits that vary among them
    k_bvhb_scatter<<<gridFor(n, smCount), 256, 0, s>>>(p);
    BVHB_CU(cudaMemsetAsync(p.cenBounds, 0xFF, 12, s)); BVHB_CU(cudaMemsetAsync(p.cenBounds + 3, 0, 12, s)); BVHB_CU(cudaMemsetAsync(p.varying, 0, 8, s));
    k_bvhb_bounds<<<gridFor(n, smCount), 256, 0, s>>>(p);
    k_bvhb_morton<<<gridFor(n, smCount), 256, 0, s>>>(p);
    BVHB_CU(readback(p.varying, 1));
    const u64 varying = host[0];
    // 2. stable LSD radix sort, 8 bits per pass; a digit that is the same for every key leaves the order as it is
    const uint tiles = (n + kRadixTile - 1) / kRadixTile;
    int cur = 0;
    for (uint shift = 0; shift < 64; shift += 8)
    {
        if (((varying >> shift) & 0xFFu) == 0) continue;
        k_bvhb_radix_hist<<<tiles, kRadixTile, 0, s>>>(p.keys[cur], n, shift, p.hist, tiles);
        launchExclusiveScan<u64>(p.hist, p.hist, 256 * tiles, scratch.scanBlocks, scratch.misc, s);
        k_bvhb_radix_scatter<<<tiles, kRadixTile, 0, s>>>(p.keys[cur], p.vals[cur], p.keys[cur ^ 1], p.vals[cur ^ 1], n, shift, p.hist, tiles);
        cur ^= 1; r.radixPasses++;
    }
    p.sorted = p.vals[cur];
    // 3. PLOC until one cluster is left
    k_bvhb_leaves<<<gridFor(n, smCount), 256, 0, s>>>(p);
    uint count = n, nextNode = n; int src = 0;
    while (count > 1)
    {
        k_bvhb_ploc_nn<<<gridFor(count, smCount), 256, 0, s>>>(p, p.clusters[src], count);
        k_bvhb_ploc_flags<<<gridFor(count, smCount), 256, 0, s>>>(p, count);
        launchExclusiveScan<u64>(p.flags, p.flags, count, scratch.scanBlocks, scratch.misc, s);
        k_bvhb_ploc_merge<<<gridFor(count, smCount), 256, 0, s>>>(p, p.clusters[src], p.clusters[src ^ 1], count, nextNode);
        BVHB_CU(readback(scratch.misc, 1));
        const uint merges = uint(host[0] >> 32), kept = uint(host[0]);
        if (merges == 0) { r.status = BvhBuildResult::kStalled; return cudaSuccess; }
        nextNode += merges; count = kept; src ^= 1; r.plocIterations++;
    }
    // 4. top-down collapse, one level per launch pair; the root is the last node made (or the single triangle)
    r.rootNode2 = n > 1 ? 2 * n - 2 : 0u;
    BVHB_CU(cudaMemcpyAsync(p.nodeRoot, &r.rootNode2, 4, cudaMemcpyHostToDevice, s));
    r.levelStart.push_back(0);
    uint first = 0, end = 1, triRunning = 0;
    for (;;)
    {
        if (r.levelStart.size() > kMaxDepth) { r.status = BvhBuildResult::kTooDeep; BVHB_CU(cudaStreamSynchronize(s)); return cudaSuccess; }
        const uint m = end - first;
        k_bvhb_collapse_count<<<gridFor(m, smCount * 2), 128, 0, s>>>(p, first, end);
        launchExclusiveScan<u64>(p.levelCounts, p.levelCounts, m, scratch.scanBlocks, scratch.misc, s);
        k_bvhb_collapse_emit<<<gridFor(m, smCount * 2), 128, 0, s>>>(p, first, end, triRunning);
        BVHB_CU(readback(scratch.misc, 1));
        r.levelStart.push_back(end);
        const uint next = uint(host[0] >> 32); triRunning += uint(host[0]);
        if (next == 0) break;
        first = end; end += next;
    }
    if (triRunning != n) { r.status = BvhBuildResult::kStalled; return cudaSuccess; }
    r.nodeCount = end;
    // 5. bottom-up encoding
    for (size_t d = r.levelStart.size() - 1; d-- > 0;)
    {
        const uint a = r.levelStart[d], b = r.levelStart[d + 1];
        k_bvhb_encode<<<gridFor(b - a, smCount * 2), 128, 0, s>>>(p, a, b);
    }
    BVHB_CU(cudaGetLastError());
    BVHB_CU(cudaMemcpyAsync(r.rootBox, p.nodeBox, 24, cudaMemcpyDeviceToHost, s));
    BVHB_CU(cudaStreamSynchronize(s)); r.syncs++;
#undef BVHB_CU
    return cudaSuccess;
}

} // namespace pt
