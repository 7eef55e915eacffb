// neeat_kernels.cu - LightsBaker's NEE-AT feedback passes (SURVEY §8f row 1) as kernels over the bodies in neeat.cuh.
//   update begin:  [snapshot copy] k_na_prefilter, k_na_p0 (warp-aggregated atomics into the per-light usage counters), k_na_proxy_counts, three-kernel exclusive scan,
//                  k_na_proxy_fill (one thread per proxy slot, binary search over the offsets)
//   update end:    k_na_p1a (half resolution), k_na_p1b, k_na_tiles (one 64-thread CTA per tile: 128 keys gathered by 128 lanes' worth of work, bitonic sort in shared memory,
//                  run lengths), k_na_clear
// All of it is integer / reservoir bookkeeping bound by HBM traffic (a few tens of bytes per pixel per pass); grids are sized by the image.  Tested on the GPU by tests/test_gpu_neeat.py; the
// bodies pass tests/test_neeat_port.py on the CPU.
#include "neeat.cuh"
#include "kernels.h"

namespace pt { namespace neeat {

#define NA_XY(WW, HH) const uint x = blockIdx.x * 16 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y; if (x >= (WW) || y >= (HH)) return

__global__ void __launch_bounds__(256) k_na_prefilter(const __grid_constant__ Params p) { NA_XY(p.W, p.H); preFilterPixel(p, int(x), int(y)); }

__global__ void __launch_bounds__(256) k_na_p0(const __grid_constant__ Params p)
{
    const uint x = blockIdx.x * 16 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y;
    const bool inside = x < p.W && y < p.H;
    const uint slot = inside ? p0Pixel(p, int(x), int(y)) : 0xFFFFFFFFu;
    // WaveMatch-style aggregation (LightsBaker.hlsl:1290-1312): one atomic per distinct light per warp
    const uint active = __ballot_sync(0xFFFFFFFFu, inside);
    if (!inside) return;
    const uint peers = __match_any_sync(active, slot);
    if ((__ffs(peers) - 1) == int(threadIdx.x + threadIdx.y * 16) % 32) atomicAdd(p.feedbackCounters + slot, uint(__popc(peers)));
}

// ComputeWeights: thread = one 32-light block (as the reference), CTA = 128 blocks whose sums thread 0 adds in index order; k_na_weight_total adds the CTAs' sums in index order
__global__ void __launch_bounds__(128) k_na_weights(const __grid_constant__ Params p)
{
    __shared__ float blockSums[128];
    const uint block = blockIdx.x * 128 + threadIdx.x;
    blockSums[threadIdx.x] = block * 32u < p.lightCount ? weightBlock(p, block) : 0.0f;
    __syncthreads();
    if (threadIdx.x == 0) { float g = 0.0f; for (int i = 0; i < 128; i++) if ((blockIdx.x * 128 + i) * 32u < p.lightCount) g = __fadd_rn(g, blockSums[i]); p.weightGroupSums[blockIdx.x] = g; }
}
__global__ void k_na_weight_total(const __grid_constant__ Params p, uint groups) { float t = 0.0f; for (uint g = 0; g < groups; g++) t = __fadd_rn(t, p.weightGroupSums[g]); *p.weightsSumDev = t; }

__global__ void __launch_bounds__(256) k_na_proxy_counts(const __grid_constant__ Params p)
{
    const uint i = blockIdx.x * 256 + threadIdx.x;
    if (i < p.lightCount) p.proxyCounters[i] = proxyCountOfLight(p, i);
}

// ---- exclusive scan of proxyCounters[0 .. lightCount) into proxyOffsets[0 .. lightCount], total into *samplingProxyCount --------------------------------------------------------
constexpr uint kScanBlock = 1024;
__device__ __forceinline__ uint blockExclusiveScan(uint v, uint* warpSums /* 32 */, uint& blockTotal)
{
    const uint lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint inc = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= uint(d)) inc += n; }
    if (lane == 31) warpSums[warp] = inc;
    __syncthreads();
    if (warp == 0)
    {
        uint w = warpSums[lane], winc = w;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint n = __shfl_up_sync(0xFFFFFFFFu, winc, d); if (lane >= uint(d)) winc += n; }
        warpSums[lane] = winc - w;                      // exclusive warp offsets
        if (lane == 31) warpSums[32] = winc;            // block total
    }
    __syncthreads();
    blockTotal = warpSums[32];
    return inc - v + warpSums[warp];
}
__global__ void __launch_bounds__(kScanBlock) k_na_scan_reduce(const __grid_constant__ Params p, uint* blockSums)
{
    __shared__ uint ws[33];
    const uint i = blockIdx.x * kScanBlock + threadIdx.x;
    uint total; blockExclusiveScan(i < p.lightCount ? p.proxyCounters[i] : 0u, ws, total);
    if (threadIdx.x == 0) blockSums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(kScanBlock) k_na_scan_blocks(const __grid_constant__ Params p, uint* blockSums, uint blockCount)
{   // one CTA: blockCount <= 1024 (lightCount <= 1 M)
    __shared__ uint ws[33];
    uint total; const uint off = blockExclusiveScan(threadIdx.x < blockCount ? blockSums[threadIdx.x] : 0u, ws, total);
    if (threadIdx.x < blockCount) blockSums[threadIdx.x] = off;
    if (threadIdx.x == 0) { *p.samplingProxyCount = total; p.proxyOffsets[p.lightCount] = total; }
}
__global__ void __launch_bounds__(kScanBlock) k_na_scan_apply(const __grid_constant__ Params p, const uint* blockSums)
{
    __shared__ uint ws[33];
    const uint i = blockIdx.x * kScanBlock + threadIdx.x;
    uint total; const uint off = blockExclusiveScan(i < p.lightCount ? p.proxyCounters[i] : 0u, ws, total);
    if (i < p.lightCount) p.proxyOffsets[i] = off + blockSums[blockIdx.x];
}
__global__ void __launch_bounds__(256) k_na_proxy_fill(const __grid_constant__ Params p)
{
    const uint total = *p.samplingProxyCount;
    for (uint slot = blockIdx.x * 256 + threadIdx.x; slot < total; slot += gridDim.x * 256) p.proxyIndices[slot] = lightOfProxySlot(p, slot);
}

__global__ void __launch_bounds__(256) k_na_p1a(const __grid_constant__ Params p) { NA_XY(p.blendedW, p.blendedH); p1aPixel(p, x, y); }
__global__ void __launch_bounds__(256) k_na_p1b(const __grid_constant__ Params p) { NA_XY(p.W, p.H); p1bPixel(p, x, y); }
__global__ void __launch_bounds__(256) k_na_clear(const __grid_constant__ Params p) { NA_XY(p.W, p.H); clearFeedbackPixel(p, x, y); }

// P2 + P3: one CTA per tile, 64 threads, two keys each
__global__ void __launch_bounds__(64) k_na_tiles(const __grid_constant__ Params p)
{
    __shared__ uint data[kLocalProxyCount];
    const uint tx = blockIdx.x, ty = blockIdx.y, t = threadIdx.x;
    data[t] = fillTileEntry(p, tx, ty, t); data[t + 64] = fillTileEntry(p, tx, ty, t + 64);
    __syncthreads();
    #pragma unroll
    for (uint k = 2; k <= kLocalProxyCount; k <<= 1)
        for (uint j = k / 2; j > 0; j /= 2) { bitonicStep(data, t, k, j); __syncthreads(); }
    const uint base = tileBaseAddress(p, tx, ty);
    p.localSamplingBuffer[base + t] = packMiniList(data[t], runLength(data, t));
    p.localSamplingBuffer[base + t + 64] = packMiniList(data[t + 64], runLength(data, t + 64));
}

} // namespace neeat

void launchNeeatUpdateBegin(const neeat::Params& p, bool preFilter, uint* scanBlockSums, int smCount, cudaStream_t s)
{
    using namespace neeat;
    const dim3 grid((p.W + 15) / 16, (p.H + 15) / 16), block(16, 16);
    cudaMemsetAsync(p.feedbackCounters, 0, (size_t(p.lightCount) + 1) * sizeof(uint), s);
    if (p.lastFrameFeedbackAvailable)
    {
        if (preFilter)
        {   // snapshot: the processed-reservoir images are free between ClearFeedbackHistory and P1b
            cudaMemcpyAsync(p.scratchWeight, p.fbWeight, size_t(p.W) * p.H * 4, cudaMemcpyDeviceToDevice, s);
            cudaMemcpyAsync(p.scratchCandidate, p.fbCandidate, size_t(p.W) * p.H * 4, cudaMemcpyDeviceToDevice, s);
            k_na_prefilter<<<grid, block, 0, s>>>(p);
        }
        k_na_p0<<<grid, block, 0, s>>>(p);
    }
    const uint weightGroups = (p.lightCount + 32 * 128 - 1) / (32 * 128);
    k_na_weights<<<weightGroups, 128, 0, s>>>(p);
    k_na_weight_total<<<1, 1, 0, s>>>(p, weightGroups);
    const uint lightBlocks = (p.lightCount + 255) / 256, scanBlocks = (p.lightCount + kScanBlock - 1) / kScanBlock;
    k_na_proxy_counts<<<lightBlocks, 256, 0, s>>>(p);
    k_na_scan_reduce<<<scanBlocks, kScanBlock, 0, s>>>(p, scanBlockSums);
    k_na_scan_blocks<<<1, kScanBlock, 0, s>>>(p, scanBlockSums, scanBlocks);
    k_na_scan_apply<<<scanBlocks, kScanBlock, 0, s>>>(p, scanBlockSums);
    k_na_proxy_fill<<<smCount * 8, 256, 0, s>>>(p);
}
void launchNeeatUpdateEnd(const neeat::Params& p, cudaStream_t s)
{
    using namespace neeat;
    const dim3 block(16, 16);
    k_na_p1a<<<dim3((p.blendedW + 15) / 16, (p.blendedH + 15) / 16), block, 0, s>>>(p);
    k_na_p1b<<<dim3((p.W + 15) / 16, (p.H + 15) / 16), block, 0, s>>>(p);
    k_na_tiles<<<dim3(p.tilesX, p.tilesY), 64, 0, s>>>(p);
    if (p.temporalFeedbackRequired) k_na_clear<<<dim3((p.W + 15) / 16, (p.H + 15) / 16), block, 0, s>>>(p);
}

} // namespace pt
