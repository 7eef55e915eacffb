// ORACLE/_ref — TEST INFRASTRUCTURE.  Known-answer generator for stochastic texture filtering: the UNMODIFIED External/Rtxtf/STFSamplerState.hlsli and
// STFSamplerStateImpl.hlsli, streamed behind ref_hlsl_shim.h by ref_stf_tu.sh, driven as RTXPT drives them (STF_SamplerState::Create, SetFilterType / SetMagMethod /
// SetSigma, Texture2DSampleLevel on one state several times).  This file is read twice: first with STF_KAT_STANDINS for the texture objects and intrinsics the headers name,
// then, after the headers, for the driver.
//   stdin:  per case 16 words: width, height, levels, filter, sigma (f32), sampler address mode (1 wrap, 3 clamp), reseedOnSample, u.xyzw (f32), then 4 fetches x (uv.x, uv.y, lambda) -> 12 more
//   stdout: per fetch 11 words: sample position uv (f32 x2), level, the value SampleLevel returned (f32 x4), the state's u afterwards (f32 x4);
//           per case 10 words: STF_ApplyAddressingMode1D of the last position's x for modes 1..5 (f32, isBorder)
#ifdef STF_KAT_STANDINS
#include <cstdio>
#include <cstdlib>
#include <vector>

#define STF_SHADER_STAGE 9                  /* STF_SHADER_STAGE_LIBRARY: the path tracer's ray-tracing shaders */
#define STF_SHADER_MODEL_MAJOR 6
#define STF_SHADER_MODEL_MINOR 6
// STF_ALLOW_WAVE_READ stays at its default (1): the magnification methods compile, and every wave / quad / derivative intrinsic they name aborts if reached (the shim's
// single-lane wave stand-ins are renamed away for these headers)
[[noreturn]] inline void stfKatUnreachable(const char* what) { std::fprintf(stderr, "ref_kat_stf: %s called\n", what); std::abort(); }
inline uint4 StfKatWaveActiveBallot(bool) { stfKatUnreachable("WaveActiveBallot"); }
inline bool StfKatIsHelperLane() { stfKatUnreachable("IsHelperLane"); }
inline uint StfKatWaveGetLaneIndex() { stfKatUnreachable("WaveGetLaneIndex"); }
template <typename T> T StfKatWaveReadLaneAt(T, uint) { stfKatUnreachable("WaveReadLaneAt"); }
template <typename T> T StfKatDdx(T) { stfKatUnreachable("ddx"); }
template <typename T> T StfKatDdy(T) { stfKatUnreachable("ddy"); }
#define WaveActiveBallot StfKatWaveActiveBallot
#define IsHelperLane StfKatIsHelperLane
#define WaveGetLaneIndex StfKatWaveGetLaneIndex
#define WaveReadLaneAt StfKatWaveReadLaneAt
#define ddx StfKatDdx
#define ddy StfKatDdy

// what the headers do with vectors beyond what the shim offers (HLSL's per-component meaning)
inline int clamp(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }
inline float2 operator+(int2 a, float s) { return float2(float(a.x) + s, float(a.y) + s); }
inline float3 operator+(int3 a, float s) { return float3(float(a.x) + s, float(a.y) + s, float(a.z) + s); }
inline float clamp(int x, float lo, float hi) { return clamp(float(x), lo, hi); }
inline float3 operator/(int3 a, float3 b) { return float3(float(a.x) / b.x, float(a.y) / b.y, float(a.z) / b.z); }
inline float2 operator*(uint2 a, float2 b) { return float2(float(a.x) * b.x, float(a.y) * b.y); }
inline float3 operator*(uint3 a, float3 b) { return float3(float(a.x) * b.x, float(a.y) * b.y, float(a.z) * b.z); }
inline float2 operator-(int a, float2 b) { return float2(float(a) - b.x, float(a) - b.y); }
inline float2 round(float2 v) { return float2(round(v.x), round(v.y)); }
inline float3 round(float3 v) { return float3(round(v.x), round(v.y), round(v.z)); }
inline float2 clamp(float2 v, int lo, int hi) { return clamp(v, float(lo), float(hi)); }
// an inout parameter given a swizzle (STF_StochasticBilinear(st, u.xy)): copy in, copy out, as HLSL passes it
int2 STF_StochasticBilinear(float2 st, float2& u);
inline int2 STF_StochasticBilinear(float2 st, swz2<float, 0, 1>& u) { float2 t(u); const int2 r = STF_StochasticBilinear(st, t); u = t; return r; }

// Texture2D (HLSL's Texture2D<float4>): GetDimensions, and SampleLevel only where STF calls it - at a texel centre of an integer level - where it returns that texel; anything else aborts.
// The texel's value names it: (x, y, level, 1).  The sampler's address mode is the driver's (wrap or clamp).
struct StfKatTexture2D
{
    uint w, h, levels;
    void GetDimensions(uint mip, uint& width, uint& height, uint& numberOfLevels) const { if (mip != 0) stfKatUnreachable("GetDimensions(mip > 0)"); width = w; height = h; numberOfLevels = levels; }
    float4 SampleLevel(SamplerState, float2 uv, float lod) const;
    float4 Load(uint3) const { stfKatUnreachable("Texture2D::Load"); }
};
struct StfKatTexture2DArray
{
    void GetDimensions(uint, uint&, uint&, uint&, uint&) const { stfKatUnreachable("Texture2DArray"); }
    float4 SampleLevel(SamplerState, float3, float) const { stfKatUnreachable("Texture2DArray"); }
    float4 Load(uint4) const { stfKatUnreachable("Texture2DArray"); }
};
struct StfKatTexture3D
{
    void GetDimensions(uint, uint&, uint&, uint&, uint&) const { stfKatUnreachable("Texture3D"); }
    float4 SampleLevel(SamplerState, float3, float) const { stfKatUnreachable("Texture3D"); }
    float4 Load(uint4) const { stfKatUnreachable("Texture3D"); }
};
struct StfKatTextureCube
{
    void GetDimensions(uint, uint&, uint&, uint&) const { stfKatUnreachable("TextureCube"); }
    float4 SampleLevel(SamplerState, float3, float) const { stfKatUnreachable("TextureCube"); }
};
#define Texture2D StfKatTexture2D
#define Texture2DArray StfKatTexture2DArray
#define Texture3D StfKatTexture3D
#define TextureCube StfKatTextureCube

static uint g_stfKatAddressMode = 1;
static float2 g_stfKatLastUV; static float g_stfKatLastLod;       // what the last SampleLevel was given
float4 StfKatTexture2D::SampleLevel(SamplerState, float2 uv, float lod) const
{
    g_stfKatLastUV = uv; g_stfKatLastLod = lod;
    if (!(lod == std::floor(lod)) || lod < 0 || lod >= float(levels)) stfKatUnreachable("SampleLevel at a fractional or missing level");
    const uint level = uint(lod), lw = std::max(1u, w >> level), lh = std::max(1u, h >> level);
    const float sx = uv.x * float(lw) - 0.5f, sy = uv.y * float(lh) - 0.5f;
    if (std::fabs(sx - std::nearbyint(sx)) > 1e-3f || std::fabs(sy - std::nearbyint(sy)) > 1e-3f) stfKatUnreachable("SampleLevel away from a texel centre");
    long x = long(std::nearbyint(sx)), y = long(std::nearbyint(sy));
    if (g_stfKatAddressMode == 3) { x = std::min(std::max(x, 0L), long(lw) - 1); y = std::min(std::max(y, 0L), long(lh) - 1); }
    else { x = ((x % long(lw)) + long(lw)) % long(lw); y = ((y % long(lh)) + long(lh)) % long(lh); }
    return float4(float(x), float(y), float(level), 1.0f);
}

#else // the driver

static float kf(uint32_t w) { float f; std::memcpy(&f, &w, 4); return f; }
static uint32_t kw(float f) { uint32_t w; std::memcpy(&w, &f, 4); return w; }

int main()
{
    std::vector<uint32_t> out;
    uint32_t in[28];
    while (std::fread(in, 4, 28, stdin) == 28)
    {
        StfKatTexture2D tex{ in[0], in[1], in[2] };
        g_stfKatAddressMode = in[5];
        // PathTracerBridgeDonut.hlsli:652-656
        STF_SamplerState s = STF_SamplerState::Create(float4(kf(in[7]), kf(in[8]), kf(in[9]), kf(in[10])));
        s.SetFilterType(in[3]);
        s.SetMagMethod(STF_MAGNIFICATION_METHOD_NONE);
        s.SetSigma(kf(in[4]));
        s.SetReseedOnSample(in[6] != 0);         // _Create leaves it unset: the driver states it
        float lastX = 0.0f; uint lastW = 1;
        for (int f = 0; f < 4; f++)
        {
            const float2 uv(kf(in[11 + 3 * f]), kf(in[12 + 3 * f]));
            const float lambda = kf(in[13 + 3 * f]);
            const float4 v = s.Texture2DSampleLevel(tex, SamplerState{}, uv, lambda);
            const uint level = uint(g_stfKatLastLod), lw = std::max(1u, tex.w >> level);
            const float4 uAfter = s.GetUniformRandom();
            out.push_back(kw(g_stfKatLastUV.x)); out.push_back(kw(g_stfKatLastUV.y)); out.push_back(level);
            out.push_back(kw(v.x)); out.push_back(kw(v.y)); out.push_back(kw(v.z)); out.push_back(kw(v.w));
            out.push_back(kw(uAfter.x)); out.push_back(kw(uAfter.y)); out.push_back(kw(uAfter.z)); out.push_back(kw(uAfter.w));
            lastX = uv.x; lastW = lw;
        }
        for (uint mode = 1; mode <= 5; mode++)
        {
            bool isBorder = false;
            const float a = STF_ApplyAddressingMode1D(lastX, lastW, mode, isBorder);
            out.push_back(kw(a)); out.push_back(isBorder ? 1u : 0u);
        }
    }
    std::fwrite(out.data(), 4, out.size(), stdout);
    return 0;
}

#endif
