// stf.cuh — stochastic texture filtering (RTXTF, External/Rtxtf/STFSamplerStateImpl.hlsli) as RTXPT reaches it with RTXPT_STOCHASTIC_TEXTURE_FILTERING_ENABLE:
// ExplicitRayConesLodTextureSampler::sampleTexture calls STF_SamplerState::Texture2DSampleLevel (Scene/Material/TextureSampler.hlsli:108-116), i.e. _Texture2DSampleImpl with
// STF_MIP_VALUE_MODE_MIP_LEVEL and, at STF_MAGNIFICATION_METHOD_NONE, no wave exchange: one stochastic integer mip, one stochastic texel of the chosen filter at that mip, and one
// fetch at that texel's centre.  __host__ __device__ so that tests/emu/stf_host_emu.cu runs the same source against the reference's headers (tests/golden/stf_golden.npz).
// The fetch itself is the caller's: the device samples a point-filtered texture object over the same mip arrays, which returns the texel exactly.
#pragma once
#include "device_math.cuh"

namespace pt {

// STFDefinitions.h
constexpr uint kStfFilterPoint = 0, kStfFilterLinear = 1, kStfFilterCubic = 2, kStfFilterGaussian = 3;
constexpr uint kStfAddressWrap = 1, kStfAddressMirror = 2, kStfAddressClamp = 3, kStfAddressBorder = 4, kStfAddressMirrorOnce = 5;

// float -> int as HLSL's int(x) after floor / round: in range the two agree with C; out of range (an infinite Gaussian offset at u.x = 0) D3D saturates, as the GPU's cvt does
PT_HD int stfToInt(float x)
{
#ifdef __CUDA_ARCH__
    return __float2int_rz(x);
#else
    if (x != x) return 0;
    if (x >= 2147483648.0f) return 2147483647;
    if (x <= -2147483648.0f) return -2147483647 - 1;
    return int(x);
#endif
}
PT_HD float stfRound(float x) { return rintf(x); }          // HLSL round: to nearest, ties to even

// STF_StochasticLinear(float, inout float): picks floor(x) or floor(x) + 1 with the fractional part as probability and re-uses u for the next decision
PT_HD int stfStochasticLinear(float coordinate, float& u)
{
    int s = stfToInt(floorf(coordinate));
    const float probabilityS = coordinate - float(s);
    if (u < probabilityS) { ++s; u /= probabilityS; }
    else u = (u - probabilityS) / (1.0f - probabilityS);
    return s;
}
// STF_GetStochasticBicubicWeights / STF_StochasticLinear(float4, float): one of the four B-spline taps
PT_HD int stfBicubicTap(float t, float u)
{
    const float t2 = t * t;
    const float w0 = (1.f / 6.f) * (-t * t2 + 3 * t2 - 3 * t + 1);
    const float w1 = (1.f / 6.f) * (3 * t * t2 - 6 * t2 + 4);
    const float w2 = (1.f / 6.f) * (-3 * t * t2 + 3 * t2 + 3 * t + 1);
    float wSum = w0;
    if (u < wSum) return 0;
    wSum += w1;
    if (u < wSum) return 1;
    wSum += w2;
    if (u < wSum) return 2;
    return 3;
}

// The sampler state of one path vertex (STF_SamplerStateImpl: the members _Texture2DSampleImpl reads at magnification method NONE)
struct StfState
{
    float4 u;                   // m_u: x, y for the texel, w for the mip
    uint filterType;            // STF_FILTER_TYPE_*
    float sigma;                // Gaussian
    bool reseedOnSample;        // m_reseedOnSample: write the consumed u back after a fetch
};
struct StfSamplePos { float2 uv; uint lod; };

// _GetTexture2DSamplePos with STF_MIP_VALUE_MODE_MIP_LEVEL (STFSamplerStateImpl.hlsli:389-456): `mipValue` is the caller's lambda, width / height / numberOfLevels the
// texture's (GetDimensions at level 0).  Returns the texel centre in UV space and the integer level; mutates the state as STF_MUTATING does.
PT_HD StfSamplePos stfTexture2DSamplePos(StfState& st, uint width, uint height, uint numberOfLevels, float2 uv, float mipValue)
{
    float4 u = st.u;
    const int maxLevel = int(numberOfLevels) - 1;
    const int ilod = stfStochasticLinear(mipValue, u.w);
    const uint lod = uint(ilod < 0 ? 0 : (ilod > maxLevel ? maxLevel : ilod));
    width = max(1u, width >> lod);
    height = max(1u, height >> lod);
    const float sx = uv.x * float(width) - 0.5f, sy = uv.y * float(height) - 0.5f;
    int ix = 0, iy = 0;
    if (st.filterType == kStfFilterPoint) { ix = stfToInt(stfRound(sx)); iy = stfToInt(stfRound(sy)); }
    else if (st.filterType == kStfFilterLinear) { ix = stfStochasticLinear(sx, u.x); iy = stfStochasticLinear(sy, u.y); }
    else if (st.filterType == kStfFilterCubic)
    {
        ix = stfToInt(floorf(sx)) - 1 + stfBicubicTap(sx - floorf(sx), u.x);
        iy = stfToInt(floorf(sy)) - 1 + stfBicubicTap(sy - floorf(sy), u.y);
    }
    else if (st.filterType == kStfFilterGaussian)
    {   // STF_StochasticGaussian2D + STF_BoxMullerTransform
        const float mag = sqrtf(-2.0f * logf(u.x));
        const float a = 2.0f * 3.14159265359f * u.y;
        const float ox = st.sigma * (mag * cosf(a)), oy = st.sigma * (mag * sinf(a));
        ix = stfToInt(stfRound(sx + ox)); iy = stfToInt(stfRound(sy + oy));
    }
    if (st.reseedOnSample) st.u = u;
    StfSamplePos r;
    r.uv = make_float2((float(ix) + 0.5f) / float(width), (float(iy) + 0.5f) / float(height));
    r.lod = lod;
    return r;
}

// STF_ApplyAddressingMode1D (STFSamplerStateImpl.hlsli:290-316): the software addressing of the Load variants; the texture objects do the sampler's wrap in hardware
PT_HD float stfApplyAddressingMode1D(float u, uint size, uint mode, bool& isBorder)
{
    const float invSize = 1.0f / float(size);
    isBorder = false;
    switch (mode)
    {
    case kStfAddressWrap:
    default:                    return u - floorf(u);
    case kStfAddressMirror:     { const float h = u * 0.5f; return 1.0f - fabsf(1.0f - (h - floorf(h)) * 2.0f); }
    case kStfAddressClamp:      return fminf(fmaxf(u, invSize), 1.0f - invSize);
    case kStfAddressBorder:     isBorder = (u <= 0.0f) || (u >= 1.0f); return fminf(fmaxf(u, invSize), 1.0f - invSize);
    case kStfAddressMirrorOnce: return fminf(fmaxf(fabsf(u), invSize), 1.0f - invSize);
    }
}

// Bridge::loadSurface (PathTracerBridgeDonut.hlsli:637-656): u from a fresh uniform generator of the vertex (SampleGeneratorVertexBase of pixel, vertex, sample; effect seed Base),
// four draws in x, y, z, w order, so that no other random stream of the vertex moves
PT_HD float4 stfVertexRandom(uint packedPixel, uint vertexIndex, uint sampleIndex)
{
    UniformSeq g = UniformSeq::make(vertexBaseHash(packedPixel, vertexIndex), sampleIndex, 0u);
    float4 u;
    u.x = g.next(); u.y = g.next(); u.z = g.next(); u.w = g.next();
    return u;
}

} // namespace pt
