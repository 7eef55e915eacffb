// refit_kernels.cu - rigid-instance animation: k_refit_tris (one thread per leaf triangle: 48 B read of the shade record's positions + 48 B rewrite of the leaf triangle) and
// k_refit_level (one thread per node of a level, deepest level first, root last: 80 B node + its children's bounds).  HBM-bound streaming passes; the number of level launches
// is the depth of the 8-wide tree (about log8 of the node count).  Tested on the GPU by tests/test_gpu_refit.py (a refitted tree traces like a fresh upload, bit for bit); the bodies also pass tests/test_refit.py on the CPU.
#include "refit.cuh"
#include "kernels.h"

namespace pt { namespace refit {

__global__ void __launch_bounds__(256) k_refit_tris(const __grid_constant__ Params p)
{
    for (uint i = blockIdx.x * 256 + threadIdx.x; i < p.triCount; i += gridDim.x * 256) refitTriangle(p, i);
}
__global__ void __launch_bounds__(128) k_refit_level(const __grid_constant__ Params p, uint first, uint end)
{
    for (uint ni = first + blockIdx.x * 128 + threadIdx.x; ni < end; ni += gridDim.x * 128) refitNode(p, ni);
}

} // namespace refit

void launchRefit(const refit::Params& p, const uint32_t* levelStart, uint32_t levelCount, int smCount, cudaStream_t s)
{
    refit::k_refit_tris<<<smCount * 8, 256, 0, s>>>(p);
    for (uint32_t d = levelCount; d-- > 0;)
    {
        const uint32_t first = levelStart[d], end = levelStart[d + 1];
        if (end > first) refit::k_refit_level<<<std::min<uint32_t>((end - first + 127) / 128, uint32_t(smCount) * 16), 128, 0, s>>>(p, first, end);
    }
}

} // namespace pt
