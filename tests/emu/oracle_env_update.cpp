// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// The oracle (oracle/oracle.cpp, compiled unchanged into this unit) plus the entry points the tests of rtxpt_b200_update_env_map need: replace a live oracle context's environment
// cube and importance map and re-bake its light list from them, read back its importance chain and lookup map, and build the importance map of a bare cube.  The result,
// tests/emu/_build/liboracle_env.so, exports every entry point of liboracle.so as well; tests/test_gpu_env_update.py loads it in its place.
#include "../../oracle/oracle.cpp"
#include <map>

namespace {
std::map<void*, std::vector<float>> g_envCubes;        // the cube each context samples after oracle_set_env_cube (the description's face pointers point into it); kept until the process ends
}

extern "C" {

// the environment was re-baked (rtxpt_b200_update_env_map): replaces the cube (allMips: the MIP chain, faces back to back per MIP, as oracle_bake_env_map returns it) and, when
// `radianceChain` is given (the 11 MIPs of the 1024^2 RGBA radiance / importance map back to back), the importance map; without it the map is built from the new cube.  Then the
// light list is re-baked from that map, and NEE-AT's next update_begin maps last frame's feedback onto it.  Call after oracle_set_constants.
ORC_API int oracle_set_env_cube(void* p, uint32_t faceSize, uint32_t mipLevels, const float* allMips, const float* radianceChain)
{
    OracleCtx* c = (OracleCtx*)p;
    if (!allMips || faceSize == 0 || mipLevels == 0 || mipLevels > RTXPT_MAX_MIPS || !c->haveConsts) return -1;
    size_t total = 0; for (uint32_t m = 0; m < mipLevels; m++) total += size_t(6) * (faceSize >> m) * (faceSize >> m) * 4;
    std::vector<float>& cube = g_envCubes[p]; cube.assign(allMips, allMips + total);
    RtxptEnvCubeDesc& e = c->descCopy.envCube; e = RtxptEnvCubeDesc{}; e.faceSize = faceSize; e.mipLevels = mipLevels;       // Scene::env points at this description
    size_t off = 0;
    for (uint32_t m = 0; m < mipLevels; m++) { const size_t face = size_t(faceSize >> m) * (faceSize >> m) * 4; for (int f = 0; f < 6; f++) { e.faces[f][m] = cube.data() + off; off += face; } }
    if (radianceChain)
    {
        LightTable& lt = c->lights; lt.importanceMipCount = firstbithigh(IMPORTANCE_MAP_DIM) + 1; lt.radianceMips.assign(lt.importanceMipCount, std::vector<float>());
        off = 0; for (uint32_t m = 0; m < lt.importanceMipCount; m++) { const size_t n = size_t(IMPORTANCE_MAP_DIM >> m) * (IMPORTANCE_MAP_DIM >> m) * 4; lt.radianceMips[m].assign(radianceChain + off, radianceChain + off + n); off += n; }
    }
    else buildEnvRadianceMap(c->scene, c->lights);
    bakeLights(c->scene, c->consts, c->lights, false);
    return 0;
}
// what: 0 the radiance / importance MIP chain (RGBA32F, MIPs back to back), 1 the environment lookup map (uint32 1024^2); returns the bytes written, or the size with out == NULL
ORC_API int64_t oracle_get_env_maps(void* p, int what, void* out, size_t bytes)
{
    OracleCtx* c = (OracleCtx*)p; const LightTable& lt = c->lights;
    size_t n = 0;
    if (what == 0) for (const std::vector<float>& m : lt.radianceMips) n += m.size() * 4;
    else if (what == 1) n = lt.envLookupMap.size() * 4;
    else return -1;
    if (!out) return int64_t(n);
    if (bytes < n) return -1;
    if (what == 1) memcpy(out, lt.envLookupMap.data(), n);
    else { size_t off = 0; for (const std::vector<float>& m : lt.radianceMips) { memcpy(static_cast<uint8_t*>(out) + off, m.data(), m.size() * 4); off += m.size() * 4; } }
    return int64_t(n);
}
// LightBaker::buildEnvRadianceMap's restatement on a bare cube (MIP 0 only, 6 faces of faceSize^2 RGBA32F): the 11 MIPs of the radiance / importance map back to back
ORC_API int oracle_env_radiance_map(uint32_t faceSize, const float* cubeMip0, float* out)
{
    if (!cubeMip0 || !out || faceSize == 0) return -1;
    RtxptEnvCubeDesc d{}; d.faceSize = faceSize; d.mipLevels = 1;
    for (int f = 0; f < 6; f++) d.faces[f][0] = cubeMip0 + size_t(f) * faceSize * faceSize * 4;
    Scene sc; sc.env.d = &d; LightTable lt;
    buildEnvRadianceMap(sc, lt);
    size_t off = 0; for (const std::vector<float>& m : lt.radianceMips) { memcpy(out + off, m.data(), m.size() * 4); off += m.size(); }
    return 0;
}

} // extern "C"
