// scan.cuh - exclusive prefix sums on the device, shared by NEE-AT's proxy offsets (neeat_kernels.cu) and the BVH builder's compactions (bvh_build_kernels.cu).
// Three kernels: per-block totals, one CTA scanning the block totals, per-block scans plus the block's offset.  Integer sums only, so the result does not depend on the launch shape.
#pragma once
#include <cuda_runtime.h>

namespace pt {

constexpr unsigned kScanBlock = 1024;

// exclusive scan of one value per thread across a CTA of kScanBlock threads; blockTotal := the CTA's sum.  warpSums: 33 entries of shared memory
template <typename T> __device__ __forceinline__ T blockExclusiveScan(T v, T* warpSums, T& blockTotal)
{
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = v;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const T n = __shfl_up_sync(0xFFFFFFFFu, inc, d); if (lane >= unsigned(d)) inc += n; }
    if (lane == 31) warpSums[warp] = inc;
    __syncthreads();
    if (warp == 0)
    {
        T w = warpSums[lane], winc = w;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const T n = __shfl_up_sync(0xFFFFFFFFu, winc, d); if (lane >= unsigned(d)) winc += n; }
        warpSums[lane] = winc - w;                      // exclusive warp offsets
        if (lane == 31) warpSums[32] = winc;            // block total
    }
    __syncthreads();
    blockTotal = warpSums[32];
    return inc - v + warpSums[warp];
}

// ---- out[i] = in[0] + ... + in[i - 1] over i < n, *total = the sum of all n (in == out allowed) ------------------------------------------------------------------------------------
template <typename T> __global__ void __launch_bounds__(kScanBlock) k_scan_reduce(const T* in, unsigned n, T* blockSums)
{
    __shared__ T ws[33];
    const unsigned i = blockIdx.x * kScanBlock + threadIdx.x;
    T total; blockExclusiveScan<T>(i < n ? in[i] : T(0), ws, total);
    if (threadIdx.x == 0) blockSums[blockIdx.x] = total;
}
template <typename T> __global__ void __launch_bounds__(kScanBlock) k_scan_blocks(T* blockSums, unsigned blockCount, T* total)
{   // one CTA, any number of blocks: kScanBlock at a time, carrying the running sum
    __shared__ T ws[33];
    T carry = 0;
    for (unsigned base = 0; base < blockCount; base += kScanBlock)
    {
        const unsigned i = base + threadIdx.x;
        T sum; const T off = blockExclusiveScan<T>(i < blockCount ? blockSums[i] : T(0), ws, sum);
        if (i < blockCount) blockSums[i] = carry + off;
        carry += sum;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = carry;
}
template <typename T> __global__ void __launch_bounds__(kScanBlock) k_scan_apply(const T* in, unsigned n, const T* blockSums, T* out)
{
    __shared__ T ws[33];
    const unsigned i = blockIdx.x * kScanBlock + threadIdx.x;
    T total; const T off = blockExclusiveScan<T>(i < n ? in[i] : T(0), ws, total);
    if (i < n) out[i] = off + blockSums[blockIdx.x];
}
// blockSums: ceil(n / kScanBlock) entries of scratch
template <typename T> inline void launchExclusiveScan(const T* in, T* out, unsigned n, T* blockSums, T* total, cudaStream_t s)
{
    const unsigned blocks = (n + kScanBlock - 1) / kScanBlock;
    if (blocks) k_scan_reduce<T><<<blocks, kScanBlock, 0, s>>>(in, n, blockSums);
    k_scan_blocks<T><<<1, kScanBlock, 0, s>>>(blockSums, blocks, total);
    if (blocks) k_scan_apply<T><<<blocks, kScanBlock, 0, s>>>(in, n, blockSums, out);
}

} // namespace pt
