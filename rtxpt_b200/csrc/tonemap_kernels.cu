// tonemap_kernels.cu - luminance reduction (grid-stride accumulation in double, block tree, then one block over the per-block partials: no atomics, deterministic) and the
// tone-mapping pass (one thread per pixel, RGBA16F or RGBA32F in, SRGBA8 out).  Streaming passes: 8-16 B read + 4 B written per pixel.  Tested on the GPU by tests/test_gpu_tonemap.py (byte-identical to the oracle in the IEEE build).
#include "tonemap.cuh"
#include "kernels.h"

namespace pt { namespace tonemap {

template <bool F32> PT_DEVICE float4 loadPixel(const void* src, size_t i)
{
    if (F32) return reinterpret_cast<const float4*>(src)[i];
    const uint2 v = reinterpret_cast<const uint2*>(src)[i];
    return make_float4(f16tof32(v.x), f16tof32(v.x >> 16), f16tof32(v.y), f16tof32(v.y >> 16));
}
constexpr int kReduceBlocks = 528;      // 132 SMs (H100 SXM) x 4
template <bool F32>
__global__ void __launch_bounds__(256) k_tm_luminance(const void* src, uint pixelCount, double* partials)
{
    __shared__ double sh[256];
    double s = 0.0;
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < pixelCount; i += gridDim.x * 256) { const float4 c = loadPixel<F32>(src, i); s += double(logLuminance(mk3(c.x, c.y, c.z))); }
    sh[threadIdx.x] = s; __syncthreads();
    for (int d = 128; d > 0; d >>= 1) { if (int(threadIdx.x) < d) sh[threadIdx.x] += sh[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}
__global__ void __launch_bounds__(1024) k_tm_finish(const double* partials, uint count, uint pixelCount, float* avgLuminance)
{
    __shared__ double sh[1024];
    sh[threadIdx.x] = threadIdx.x < count ? partials[threadIdx.x] : 0.0; __syncthreads();
    for (int d = 512; d > 0; d >>= 1) { if (int(threadIdx.x) < d) sh[threadIdx.x] += sh[threadIdx.x + d]; __syncthreads(); }
    if (threadIdx.x == 0) *avgLuminance = exp2f(float(sh[0] / double(pixelCount)));
}
template <bool F32>
__global__ void __launch_bounds__(256) k_tm_apply(const __grid_constant__ Params p, const void* src, uint pixelCount, const float* avgLuminance, uint* dst)
{
    const uint i = blockIdx.x * 256 + threadIdx.x;
    if (i >= pixelCount) return;
    const float4 c = loadPixel<F32>(src, i);
    dst[i] = packLdr(applyToneMapping(p, p.autoExposure ? *avgLuminance : 1.0f, mk3(c.x, c.y, c.z)), c.w);
}

} // namespace tonemap

void launchToneMap(const tonemap::Params& p, const void* src, bool srcIsF32, uint32_t pixelCount, double* partials, float* avgLuminance, uint32_t* dst, cudaStream_t s)
{
    using namespace tonemap;
    if (srcIsF32) k_tm_luminance<true><<<kReduceBlocks, 256, 0, s>>>(src, pixelCount, partials); else k_tm_luminance<false><<<kReduceBlocks, 256, 0, s>>>(src, pixelCount, partials);
    k_tm_finish<<<1, 1024, 0, s>>>(partials, kReduceBlocks, pixelCount, avgLuminance);
    if (srcIsF32) k_tm_apply<true><<<(pixelCount + 255) / 256, 256, 0, s>>>(p, src, pixelCount, avgLuminance, dst); else k_tm_apply<false><<<(pixelCount + 255) / 256, 256, 0, s>>>(p, src, pixelCount, avgLuminance, dst);
}

} // namespace pt
