// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of the importance-map bodies rtxpt_b200_update_env_map runs on the GPU (rtxpt_b200/csrc/envbake.cuh: importanceTexel, importanceReduceTexel), in
// launchEnvImportance's order.  tests/test_env_update.py holds it to the oracle's buildEnvRadianceMap bit for bit; libdevice's cos / sin stay with tests/test_gpu_env_update.py.
#include "../../rtxpt_b200/csrc/envbake.cuh"
#include <cstdint>

// cube: MIP 0, 6 faces of faceSize^2 RGBA32F; out: the 11 MIPs of the 1024^2 RGBA map back to back
extern "C" int emu_env_importance_map(uint32_t faceSize, const float* cube, float* out)
{
    using namespace pt::envbake;
    if (!cube || !out || faceSize == 0) return -1;
    ImportanceParams p{}; p.cube = cube; p.faceSize = faceSize;
    size_t off = 0; for (uint32_t m = 0; m < kImportanceMips; m++) { p.mips[m] = out + off; off += size_t(kImportanceDim >> m) * (kImportanceDim >> m) * 4; }
    #pragma omp parallel for schedule(dynamic, 8)
    for (int y = 0; y < int(kImportanceDim); y++) for (uint32_t x = 0; x < kImportanceDim; x++) importanceTexel(p, x, uint32_t(y));
    for (uint32_t m = 1; m < kImportanceMips; m++) { const uint32_t n = kImportanceDim >> m; for (uint32_t y = 0; y < n; y++) for (uint32_t x = 0; x < n; x++) importanceReduceTexel(p, m, x, y); }
    return 0;
}
