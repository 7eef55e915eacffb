// skinning_kernels.cu - k_skin_vertices (Donut's skinning_cs: one thread per vertex) and k_skin_gather (one thread per triangle: skinned vertices -> the path tracer's per-triangle
// shade records).  Streaming passes over one geometry; the BVH refit follows (rtxpt_b200_update_instance_transforms).  Tested on the GPU by tests/test_gpu_skinning.py (every word of the rewritten shade records
// and the previous-position ranges equal the oracle's skin: 203 k vertices, 64 joints, four weights, normals and tangents; offset geometries, instancing, several skins) and tests/test_motion_vectors.py.
#include "skinning.cuh"
#include "kernels.h"

namespace pt { namespace skin {
__global__ void __launch_bounds__(256) k_skin_vertices(const __grid_constant__ Params p) { const uint i = blockIdx.x * 256 + threadIdx.x; if (i < p.numVertices) skinVertex(p, i); }
__global__ void __launch_bounds__(256) k_skin_gather(const __grid_constant__ Params p) { const uint t = blockIdx.x * 256 + threadIdx.x; if (t < p.numTriangles) gatherTriangle(p, t); }
__global__ void __launch_bounds__(256) k_skin_init_prev(const __grid_constant__ Params p) { const uint t = blockIdx.x * 256 + threadIdx.x; if (t < p.numTriangles) initPrevTriangle(p, t); }
} // namespace skin
void launchSkinInitPrev(const skin::Params& p, cudaStream_t s) { if (p.numTriangles) skin::k_skin_init_prev<<<(p.numTriangles + 255) / 256, 256, 0, s>>>(p); }
void launchSkin(const skin::Params& p, cudaStream_t s)
{
    if (p.numVertices) skin::k_skin_vertices<<<(p.numVertices + 255) / 256, 256, 0, s>>>(p);
    if (p.numTriangles) skin::k_skin_gather<<<(p.numTriangles + 255) / 256, 256, 0, s>>>(p);
}
} // namespace pt
