// envbake_kernels.cu - EnvMapBaker's BaseLayerCS and MIPReduceCS over the bodies in envbake.cuh: one thread per half-resolution texel and face, 8x8 CTAs as the reference
// dispatches them.  A bake is a once-per-environment-change job (a 2048 cube: 25 M source taps, ~0.5 GB written), bound by the transcendental maths of the direction / solid
// angle functions rather than by HBM.  Tested on the GPU by tests/test_gpu_envbake.py; the bodies also pass tests/test_envbake.py on the CPU.
#include "envbake.cuh"
#include "kernels.h"

namespace pt { namespace envbake {

__global__ void __launch_bounds__(64) k_eb_base_layer(const __grid_constant__ Params p, uint hasMip1)
{
    const uint x = blockIdx.x * 8 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, half = p.cubeDim / 2;
    if (x < half && y < half) baseLayerTexel(p, x, y, blockIdx.z, hasMip1 != 0);
}
__global__ void __launch_bounds__(64) k_eb_mip_reduce(const __grid_constant__ Params p, uint mip)
{
    const uint x = blockIdx.x * 8 + threadIdx.x, y = blockIdx.y * 8 + threadIdx.y, n = p.cubeDim >> mip;
    if (x < n && y < n) mipReduceTexel(p, mip, x, y, blockIdx.z);
}
// BuildMIPDescentImportanceMapCS: one texel of the 1024^2 map per thread, 16x16 CTAs as the reference dispatches it; 16 bilinear taps of the cube's MIP 0 each
__global__ void __launch_bounds__(256) k_eb_importance(const __grid_constant__ ImportanceParams p)
{
    const uint x = blockIdx.x * 16 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y;
    if (x < kImportanceDim && y < kImportanceDim) importanceTexel(p, x, y);
}
__global__ void __launch_bounds__(256) k_eb_importance_reduce(const __grid_constant__ ImportanceParams p, uint mip)
{
    const uint x = blockIdx.x * 16 + threadIdx.x, y = blockIdx.y * 16 + threadIdx.y, n = kImportanceDim >> mip;
    if (x < n && y < n) importanceReduceTexel(p, mip, x, y);
}

} // namespace envbake

void launchEnvBake(const envbake::Params& p, uint32_t mipLevels, cudaStream_t s)
{
    const uint32_t half = p.cubeDim / 2;
    envbake::k_eb_base_layer<<<dim3((half + 7) / 8, (half + 7) / 8, 6), dim3(8, 8), 0, s>>>(p, mipLevels > 1 ? 1u : 0u);
    for (uint32_t m = 2; m < mipLevels; m++) { const uint32_t n = p.cubeDim >> m; envbake::k_eb_mip_reduce<<<dim3((n + 7) / 8, (n + 7) / 8, 6), dim3(8, 8), 0, s>>>(p, m); }
}
void launchEnvImportance(const envbake::ImportanceParams& p, cudaStream_t s)
{
    using namespace envbake;
    k_eb_importance<<<dim3(kImportanceDim / 16, kImportanceDim / 16), dim3(16, 16), 0, s>>>(p);
    for (uint32_t m = 1; m < kImportanceMips; m++) { const uint32_t n = kImportanceDim >> m; k_eb_importance_reduce<<<dim3((n + 15) / 16, (n + 15) / 16), dim3(16, 16), 0, s>>>(p, m); }
}

} // namespace pt
