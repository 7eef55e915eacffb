// ORACLE/_ref — TEST INFRASTRUCTURE.  Known-answer generator for RTXPT's DLSS-RR input pass: the UNMODIFIED PostProcess.hlsl (ComputeSpecularMotionVector, :94-160, and the
// DENOISER_DLSS_RR main, :175-440) compiled in place behind ref_hlsl_shim.h and the path-tracer headers of ref_hlsl_tu.sh, streamed by ref_dlss_rr_tu.sh.  This file is read
// twice: first (DLSS_RR_KAT_DRIVER undefined) for the stand-ins of what the pass reads beyond those headers, then, after the pass, for the driver.
//   stdin:  per record 104 words (tests/golden/make_dlss_rr_golden.py):
//     0 active stable plane count, 1 DLSSRRBrightnessClampK (f32), 2-5 the pixel's stable-plane header (branch IDs of planes 0-2, first-hit length | dominant index),
//     6-65 the three StablePlane records (20 words each, RtxptStablePlane layout), 66-67 stable radiance (RGBA16F), 68 u_SpecularHitT (f32), 69 u_MotionVectors.xy (RG16F),
//     70-85 view.matWorldToClipNoOffset, 86-101 previousView.matWorldToClipNoOffset (row-major, f32), 102-103 view.clipToWindowScale (f32)
//   stdout: per record 15 floats, the values the pass stores before the targets' format conversion: u_OutputColor.rgb, u_RRDiffuseAlbedo.rgb, u_RRSpecAlbedo.rgb,
//     u_RRNormalsAndRoughness.xyzw, u_RRSpecMotionVectors.xy
#ifndef DLSS_RR_KAT_DRIVER
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <vector>
// float4x4 and the row-vector mul of SampleConstantBuffer.h's PlanarViewConstants (#pragma pack_matrix(row_major), PostProcess.hlsl:14)
struct ShimFloat4x4 { float m[4][4]; };
typedef ShimFloat4x4 float4x4;
inline float4 mul(float4 v, const float4x4& M)
{
    float r[4];
    for (int c = 0; c < 4; c++) r[c] = v.x * M.m[0][c] + v.y * M.m[1][c] + v.z * M.m[2][c] + v.w * M.m[3][c];
    return float4(r[0], r[1], r[2], r[3]);
}
// g_Const (SampleConstants): the members the pass reads
struct ShimPlanarView { float4x4 matWorldToClipNoOffset; float2 clipToWindowScale; };
struct ShimSampleConstants { PathTracerConstants ptConsts; ShimPlanarView view, previousView; DebugConstants debug; };
static ShimSampleConstants g_Const;
// the u_* views of ShaderResourceBindings.hlsli
static RWTexture2DArray<uint> u_StablePlanesHeader; static RWStructuredBuffer<StablePlane> u_StablePlanesBuffer; static RWTexture2D<float4> u_StableRadiance;
static RWTexture2D<float> u_SpecularHitT; static RWTexture2D<float4> u_MotionVectors, u_Depth, u_OutputColor, u_RRDiffuseAlbedo, u_RRSpecAlbedo, u_RRNormalsAndRoughness;
static RWTexture2D<float2> u_RRSpecMotionVectors;
struct ShimHalfResTexture { void GetDimensions(uint& w, uint& h) const { w = h = 1; } float4 operator[](int2) const { return float4(0, 0, 0, 0); } };
static ShimHalfResTexture u_DenoisingAvgLayerRadiance;         // read only by SampleAvgLayerRadiance, whose call is compiled out (#if 0, :235)
static RWStructuredBuffer<DebugFeedbackStruct> u_FeedbackBuffer; static RWStructuredBuffer<DebugLineStruct> u_DebugLinesBuffer;
static RWStructuredBuffer<DeltaTreeVizPathVertex> u_DebugDeltaPathTree; static RWStructuredBuffer<PathPayload> u_DeltaPathSearchStack;
inline void DebugPixel(uint2, float4) {}                      // the debug overlays are off (ENABLE_DEBUG_VIZUALISATIONS 0)
float4 (*g_shimCubeSample)(float3 dir, float lod) = nullptr;   // the shim's environment-cube hook: the path-tracer headers name it, this pass never samples it
#else
int main()
{
    std::vector<uint32_t> in; uint32_t w;
    while (std::fread(&w, 4, 1, stdin) == 1) in.push_back(w);
    const int kIn = 104;
    // a 1 x 1 image: GenericTS addressing still pads it to one 8 x 8 tile per plane
    uint header[4]; StablePlane planes[3 * 64]; float4 stableRadiance, motion, outColor, diffAlbedo, specAlbedo, normalsRoughness; float specHitT; float2 specMotion;
    u_StablePlanesHeader.p = header; u_StablePlanesHeader.w = u_StablePlanesHeader.h = 1; u_StablePlanesHeader.d = 4;
    u_StablePlanesBuffer.p = planes; u_StablePlanesBuffer.n = 3 * 64;
    auto bind = [](auto& view, auto* p) { view.p = p; view.w = view.h = 1; };
    bind(u_StableRadiance, &stableRadiance); bind(u_SpecularHitT, &specHitT); bind(u_MotionVectors, &motion); bind(u_OutputColor, &outColor);
    bind(u_RRDiffuseAlbedo, &diffAlbedo); bind(u_RRSpecAlbedo, &specAlbedo); bind(u_RRNormalsAndRoughness, &normalsRoughness); bind(u_RRSpecMotionVectors, &specMotion);
    for (size_t i = 0; i + kIn <= in.size(); i += kIn)
    {
        const uint32_t* r = &in[i];
        memset(&g_Const.ptConsts, 0, sizeof(g_Const.ptConsts));
        g_shimActivePlaneCount = r[0];
        g_Const.ptConsts.imageWidth = g_Const.ptConsts.imageHeight = 1;
        g_Const.ptConsts.genericTSLineStride = GenericTSComputeLineStride(1, 1); g_Const.ptConsts.genericTSPlaneStride = GenericTSComputePlaneStride(1, 1);
        g_Const.ptConsts.DLSSRRBrightnessClampK = asfloat(r[1]);
        for (int k = 0; k < 4; k++) header[k] = r[2 + k];
        memset(planes, 0, sizeof(planes));
        for (uint k = 0; k < 3; k++)
        {
            const uint32_t* s = r + 6 + 20 * k; StablePlane& sp = planes[GenericTSPixelToAddress(uint2(0, 0), k, g_Const.ptConsts.genericTSLineStride, g_Const.ptConsts.genericTSPlaneStride)];
            sp.RayOrigin = float3(asfloat(s[0]), asfloat(s[1]), asfloat(s[2])); sp.LastRayTCurrent = asfloat(s[3]); sp.RayDir = float3(asfloat(s[4]), asfloat(s[5]), asfloat(s[6])); sp.SceneLength = asfloat(s[7]);
            sp.PackedThpAndMVs = uint3(s[8], s[9], s[10]); sp.VertexIndexAndRoughness = s[11]; sp.DenoiserPackedBSDFEstimate = uint3(s[12], s[13], s[14]); sp.PackedNormal = s[15];
            sp.PackedNoisyRadianceAndSpecAvg = uint2(s[16], s[17]); sp.FlagsAndVertexIndex = s[18]; sp.PackedCounters = s[19];
        }
        stableRadiance = float4(f16tof32(r[66] & 0xFFFF), f16tof32(r[66] >> 16), f16tof32(r[67] & 0xFFFF), f16tof32(r[67] >> 16));
        specHitT = asfloat(r[68]);
        motion = float4(f16tof32(r[69] & 0xFFFF), f16tof32(r[69] >> 16), 0.0f, 0.0f);
        for (int k = 0; k < 16; k++) { g_Const.view.matWorldToClipNoOffset.m[k / 4][k % 4] = asfloat(r[70 + k]); g_Const.previousView.matWorldToClipNoOffset.m[k / 4][k % 4] = asfloat(r[86 + k]); }
        g_Const.view.clipToWindowScale = float2(asfloat(r[102]), asfloat(r[103]));
        DlssRrPrepareInputsMain(uint3(0, 0, 0));
        const float out[15] = { outColor.x, outColor.y, outColor.z, diffAlbedo.x, diffAlbedo.y, diffAlbedo.z, specAlbedo.x, specAlbedo.y, specAlbedo.z,
                                normalsRoughness.x, normalsRoughness.y, normalsRoughness.z, normalsRoughness.w, specMotion.x, specMotion.y };
        std::fwrite(out, 4, 15, stdout);
    }
    return 0;
}
#endif
