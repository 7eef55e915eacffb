// ORACLE — test infrastructure only (see pt_math.h).
// Stochastic texture filtering as RTXPT's material fetches run it with RTXPT_STOCHASTIC_TEXTURE_FILTERING_ENABLE = 1: Bridge::loadSurface makes one STF_SamplerState per vertex
// (PathTracerBridgeDonut.hlsli:637-656: u = four draws of a fresh uniform generator of (pixel, vertex, sample), filter / magnification / sigma from the constants), and every
// material fetch runs STF_SamplerState::Texture2DSampleLevel at the ray-cone lambda (TextureSampler.hlsli:108-116) on its own copy of that state (the bridge's sampleTexture takes
// the sampler by value, BridgeDonut:269-278).  _Texture2DSampleImpl at STF_MAGNIFICATION_METHOD_NONE (External/Rtxtf/STFSamplerStateImpl.hlsli:389-456, :857-887): a stochastic
// integer mip, one texel of the filter at that mip, SampleLevel at the texel's centre - which the software texture here answers with the texel itself.
// Written from the header, independently of rtxpt_b200/csrc/stf.cuh; tests/golden/stf_golden.npz holds both to the header's own compiled code.
// Used by the oracle that oracle/stf.mk writes (stf_oracle.py); the committed oracle does not include it.
#pragma once
#include "pt_rng.h"

namespace orc {

struct StfSettings { uint enable = 0, filterType = 0; float sigma = 0.3f; };     // rtxpt_b200_set_texture_filtering (magnification method NONE)

// the sampler state of the vertex whose material is being sampled (set around sampleGeometryMaterial by loadSurface; each fetch copies it)
struct StfVertexState { bool active = false; uint filterType = 0; float sigma = 0; float u[4] = {0, 0, 0, 0}; };
inline StfVertexState& stfCurrentVertex() { static thread_local StfVertexState s; return s; }
struct StfVertexScope
{
    StfVertexScope(const StfSettings& st, uint pixelX, uint pixelY, uint vertexIndex, uint sampleIndex)
    {
        StfVertexState& v = stfCurrentVertex();
        v.active = st.enable != 0;
        if (!v.active) return;
        UniformSampleSequenceGenerator g = UniformSampleSequenceGenerator::make(SampleGeneratorVertexBase::make((pixelX << 16) | pixelY, vertexIndex, sampleIndex), SeedBase);
        for (int i = 0; i < 4; i++) v.u[i] = g.Next1D();                                 // sampleNext4D: x, y, z, w in order
        v.filterType = st.filterType; v.sigma = st.sigma;
    }
    ~StfVertexScope() { stfCurrentVertex().active = false; }
};

// STF_StochasticLinear(float, inout float)
inline int stfLinearPick(float x, float& u)
{
    int s = int(floorf(x));
    const float p = x - float(s);
    if (u < p) { s += 1; u = u / p; } else u = (u - p) / (1 - p);
    return s;
}
// STF_GetStochasticBicubicWeights + STF_StochasticLinear(float4, float)
inline int stfCubicPick(float t, float u)
{
    const float t2 = t * t;
    const float w[3] = { (1.f / 6.f) * (-t * t2 + 3 * t2 - 3 * t + 1), (1.f / 6.f) * (3 * t * t2 - 6 * t2 + 4), (1.f / 6.f) * (-3 * t * t2 + 3 * t2 + 3 * t + 1) };
    float acc = 0;
    for (int i = 0; i < 3; i++) { acc += w[i]; if (u < acc) return i; }
    return 3;
}
// HLSL int(round(x)): ties to even; out of range saturates as D3D's conversion does
inline int stfRoundToInt(float x)
{
    const float r = std::nearbyint(x);
    if (r != r) return 0;
    if (r >= 2147483648.0f) return 2147483647;
    if (r <= -2147483648.0f) return -2147483647 - 1;
    return int(r);
}

// Texture2DSampleLevel(tex, s, uv, lambda) on a copy of the vertex's state: the texel at the chosen position (wrap, as s_MaterialSampler)
template <typename Texture2DT>
inline float4 stfSampleLevel(const Texture2DT& t, float2 uv, float lambda, const StfVertexState& vs)
{
    float u[4] = { vs.u[0], vs.u[1], vs.u[2], vs.u[3] };
    const int maxLevel = int(t.d->mipLevels) - 1;
    int ilod = stfLinearPick(lambda, u[3]);
    const uint lod = uint(std::min(std::max(ilod, 0), maxLevel));
    const uint w = std::max(1u, t.d->width >> lod), h = std::max(1u, t.d->height >> lod);
    const float sx = uv.x * float(w) - 0.5f, sy = uv.y * float(h) - 0.5f;
    int ix = 0, iy = 0;
    switch (vs.filterType)
    {
    case 0: ix = stfRoundToInt(sx); iy = stfRoundToInt(sy); break;
    case 1: ix = stfLinearPick(sx, u[0]); iy = stfLinearPick(sy, u[1]); break;
    case 2: ix = int(floorf(sx)) - 1 + stfCubicPick(sx - floorf(sx), u[0]); iy = int(floorf(sy)) - 1 + stfCubicPick(sy - floorf(sy), u[1]); break;
    default:
    {   // STF_BoxMullerTransform, STF_StochasticGaussian2D
        const float mag = sqrtf(-2.0f * logf(u[0]));
        const float angle = 2.0f * 3.14159265359f * u[1];
        ix = stfRoundToInt(sx + vs.sigma * (mag * cosf(angle))); iy = stfRoundToInt(sy + vs.sigma * (mag * sinf(angle)));
    }
    }
    // SampleLevel at ((i + 0.5) / size, lod) with a point-exact answer: the texel floor(uv * size) of that level, wrapped
    const float px = (float(ix) + 0.5f) / float(w), py = (float(iy) + 0.5f) / float(h);
    return t.texel(lod, int(floorf(px * float(w))), int(floorf(py * float(h))));
}

} // namespace orc
