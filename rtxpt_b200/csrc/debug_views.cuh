// debug_views.cuh — RTXPT's debug views (m_ui.DebugView -> DebugConstants::debugViewType, DebugViewType in PathTracer/PathTracerDebug.hlsli:25-65): the pixel colour of
// each view this library renders, from the values the path tracer already holds.  __host__ __device__ so that tests/emu/debug_views_host_emu.cu runs the same source on the CPU.
//   first hit:     surfaceDebugViz (PathTracerBridgeDonut.hlsli:457-510), from the surface the vertex-1 surface load produced
//   stable planes: StablePlanesDebugViz (PathTracerDebug.hlsli:359-461), from one plane record, the pixel's dominant plane index and its stable radiance
// The mouse-cursor crosshair and digits StablePlanesDebugViz draws on top are host UI and are not drawn.
#pragma once
#include "device_math.cuh"
#include "../../include/rtxpt_b200.h"

namespace pt {

// DebugViewType (PathTracerDebug.hlsli:25-65), the values of RTXPT_DEBUG_VIEW_* in include/rtxpt_b200.h
constexpr uint kDbgDominantStablePlaneIndex = 1, kDbgStablePlaneVirtualRayLength = 2, kDbgStablePlaneMotionVectors = 3, kDbgStablePlaneNormals = 4,
               kDbgStablePlaneRoughness = 5, kDbgStablePlaneSpecAvg = 6, kDbgStablePlaneDiffBSDFEstimate = 7, kDbgStablePlaneDiffRadiance = 8, kDbgStablePlaneSpecBSDFEstimate = 9,
               kDbgStablePlaneSpecRadiance = 10, kDbgStablePlaneRelaxedDisocclusion = 11, kDbgStablePlaneDiffRadianceDenoised = 12, kDbgStablePlaneSpecRadianceDenoised = 13,
               kDbgStablePlaneCombinedRadianceDenoised = 14, kDbgStablePlaneViewZ = 15, kDbgStablePlaneThroughput = 16, kDbgStablePlaneDenoiserValidation = 17, kDbgStableRadiance = 18,
               kDbgFirstHitBarycentrics = 29, kDbgFirstHitFaceNormal = 30, kDbgFirstHitGeometryNormal = 31, kDbgFirstHitShadingNormal = 32, kDbgFirstHitShadingTangent = 33,
               kDbgFirstHitShadingBitangent = 34, kDbgFirstHitFrontFacing = 35, kDbgFirstHitThinSurface = 36, kDbgFirstHitDiffuse = 37, kDbgFirstHitSpecular = 38,
               kDbgFirstHitRoughness = 39, kDbgFirstHitMetallic = 40, kDbgFirstHitShaderID = 41, kDbgFirstHitMaterialID = 42;

PT_HD bool isFirstHitView(uint v) { return v >= kDbgFirstHitBarycentrics && v <= kDbgFirstHitMaterialID; }
// the views StablePlanesDebugViz draws (PathTracerDebug.hlsli:362-363; Sample.cpp:2551 runs it after the FILL pass)
PT_HD bool isStablePlaneView(uint v) { return (v >= kDbgDominantStablePlaneIndex && v <= kDbgStablePlaneSpecRadiance) || v == kDbgStableRadiance; }
// the views DENOISER_FINAL_MERGE draws (PostProcess.hlsl:633-681), one stable plane per merge
PT_HD bool isDenoiserMergeView(uint v) { return v >= kDbgStablePlaneRelaxedDisocclusion && v <= kDbgStablePlaneDenoiserValidation; }

// DbgShowNormalSRGB (PathTracerShared.h:144-147): pow(abs(n * 0.5 + 0.5), 2.2).  HLSL leaves pow's precision to the compiler; here it is taken in double and rounded once to
// float, so that the device and the host agree on every value that is not within a double's error of a float rounding boundary
PT_HD float dbgPow22(float x) { return float(pow(double(x), double(2.2f))); }
PT_HD float3 dbgShowNormalSRGB(float3 n)
{
    const float3 a = n * 0.5f + mk3(0.5f);
    return mk3(dbgPow22(fabsf(a.x)), dbgPow22(fabsf(a.y)), dbgPow22(fabsf(a.z)));
}

// ColorFromHash (Utils/Utils.hlsli:109-112) over Unpack_R11G11B10_FLOAT (Utils/Packing.hlsli:186-192); saturate takes an unpacked NaN to 0 and infinity to 1
PT_HD float3 unpackR11G11B10(uint rgb) { return mk3(f16tof32((rgb << 4) & 0x7FF0u), f16tof32((rgb >> 7) & 0x7FF0u), f16tof32((rgb >> 17) & 0x7FE0u)); }
PT_HD float3 colorFromHash(uint hash) { return sat3(unpackR11G11B10(hash)); }

// GradientHeatMap (Utils/Utils.hlsli:92-107; shadertoy llKGWG): a grey value in [0, 1] to a blue-green-red heat map
PT_HD float dbgSmoothstep(float a, float b, float x) { const float t = sat((x - a) / (b - a)); return t * t * (3.0f - 2.0f * t); }      // HLSL smoothstep
PT_HD float3 gradientHeatMap(float grey)
{
    grey = sat(grey);
    float3 heat; heat.x = dbgSmoothstep(0.5f, 0.8f, grey);
    if (grey >= 0.90f) heat.x *= (1.1f - grey) * 5.0f;
    if (grey > 0.7f) heat.y = dbgSmoothstep(1.0f, 0.7f, grey);
    else heat.y = dbgSmoothstep(0.0f, 0.7f, grey);
    heat.z = dbgSmoothstep(1.0f, 0.0f, grey);
    if (grey <= 0.3f) heat.z *= grey / 0.3f;
    return heat;
}

// StablePlaneDebugVizColor (StablePlanes.hlsli:314-317)
PT_HD float3 stablePlaneDebugVizColor(uint planeIndex)
{
    return mk3((planeIndex == 0 || planeIndex == 3) ? 1.0f : 0.0f, planeIndex == 1 ? 1.0f : 0.0f, (planeIndex == 2 || planeIndex == 3) ? 1.0f : 0.0f);
}
// StablePlaneDebugVizFourWaySplitCoord (StablePlanes.hlsli:321-335): a negative plane index shows the three planes (and a fourth, empty, quadrant) at half resolution
PT_HD void stablePlaneFourWaySplitCoord(int dbgPlaneIndex, uint px, uint py, uint width, uint height, uint& outX, uint& outY, uint& outPlane)
{
    if (dbgPlaneIndex >= 0) { outX = px; outY = py; outPlane = uint(dbgPlaneIndex); return; }
    const uint hx = width / 2, hy = height / 2;
    const uint qx = px >= hx ? 1u : 0u, qy = py >= hy ? 1u : 0u;
    outX = uint(float(px - qx * hx) * 2.0f); outY = uint(float(py - qy * hy) * 2.0f);
    outPlane = qx + qy * 2u;
}

// what surfaceDebugViz reads of the first hit: ShadingData and StandardBSDFData after the surface load, the hit's barycentrics and material index
struct FirstHitDebugInputs
{
    float2 barycentrics;
    float3 faceN, vertexN, N, T, B;         // ShadingData::faceNCorrected, vertexN, N, T, B
    bool frontFacing, thin;
    float3 diffuse, specular; float roughness, metallic;
    uint materialID;
};
// one pixel of a first-hit view (PathTracerBridgeDonut.hlsli:490-506).  This library has one shader for every material, as RTXPT without RTXPT_SHADER_ID: shader ID 0xFFFFFFFF
PT_HD float4 firstHitDebugColor(uint view, const FirstHitDebugInputs& s)
{
    float3 c = mk3(0.0f);
    switch (view)
    {
    case kDbgFirstHitBarycentrics:     return make_float4(s.barycentrics.x, s.barycentrics.y, 0.0f, 1.0f);
    case kDbgFirstHitFaceNormal:       c = dbgShowNormalSRGB(s.faceN); break;
    case kDbgFirstHitGeometryNormal:   c = dbgShowNormalSRGB(s.vertexN); break;
    case kDbgFirstHitShadingNormal:    c = dbgShowNormalSRGB(s.N); break;
    case kDbgFirstHitShadingTangent:   c = dbgShowNormalSRGB(s.T); break;
    case kDbgFirstHitShadingBitangent: c = dbgShowNormalSRGB(s.B); break;
    case kDbgFirstHitFrontFacing:      c = sat3(mk3(0.15f, 0.1f + (s.frontFacing ? 1.0f : 0.0f), 0.15f)); break;
    case kDbgFirstHitThinSurface:      c = sat3(mk3(0.15f, 0.1f + (s.thin ? 1.0f : 0.0f), 0.15f)); break;
    case kDbgFirstHitDiffuse:          c = s.diffuse; break;
    case kDbgFirstHitSpecular:         c = s.specular; break;
    case kDbgFirstHitRoughness:        c = mk3(s.roughness); break;
    case kDbgFirstHitMetallic:         c = mk3(s.metallic); break;
    case kDbgFirstHitShaderID:         c = colorFromHash(hash32(0xFFFFFFFFu)); break;
    case kDbgFirstHitMaterialID:       c = colorFromHash(hash32(s.materialID)); break;
    default: return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    return make_float4(c.x, c.y, c.z, 1.0f);
}

PT_HD float dbgFrac(float x) { return x - floorf(x); }        // HLSL frac
PT_HD void unpackTwoHalves(const uint32_t w[3], float3& hi, float3& lo)     // UnpackTwoFp32ToFp16 (Utils/Packing.hlsli:197)
{
    hi = mk3(f16tof32(w[0] >> 16), f16tof32(w[1] >> 16), f16tof32(w[2] >> 16)); lo = mk3(f16tof32(w[0]), f16tof32(w[1]), f16tof32(w[2]));
}

// one pixel of a StablePlanesDebugViz view (PathTracerDebug.hlsli:369-420).  branchID and sp: the plane the four-way split picked for this pixel (stablePlaneFourWaySplitCoord
// for the per-plane views, plane 0 of the pixel itself for the others); dominantIndex and stableRadiance: the pixel's own.  Alpha 0: nothing is drawn
PT_HD float4 stablePlaneDebugColor(uint view, uint px, uint py, uint branchID, const RtxptStablePlane& sp, uint dominantIndex, float3 stableRadiance)
{
    if (branchID == 0xFFFFFFFFu) { const float c = float((px + py) % 2u); return make_float4(c, c, c, 1.0f); }     // checkerboard: no plane here
    const float sceneLength = sp.SceneLength;
    float3 thp, mv; unpackTwoHalves(sp.PackedThpAndMVs, thp, mv);
    float3 diffEstimate, specEstimate; unpackTwoHalves(sp.DenoiserPackedBSDFEstimate, diffEstimate, specEstimate);
    // StablePlane::GetNoisyRadianceAndSpecRA / GetNoisyDiffRadiance / GetNoisySpecRadiance (StablePlanes.hlsli:63-69, kSpecHeuristicBoost = 1)
    const float4 l = make_float4(f16tof32(sp.PackedNoisyRadianceAndSpecAvg[0]), f16tof32(sp.PackedNoisyRadianceAndSpecAvg[0] >> 16),
                                 f16tof32(sp.PackedNoisyRadianceAndSpecAvg[1]), f16tof32(sp.PackedNoisyRadianceAndSpecAvg[1] >> 16));
    const float3 rad = mk3(l.x, l.y, l.z);
    const float totalAvg = average(rad);
    float3 c;
    switch (view)
    {
    case kDbgDominantStablePlaneIndex:    c = stablePlaneDebugVizColor(dominantIndex); break;
    case kDbgStablePlaneVirtualRayLength: c = (sceneLength >= kMaxRayTravel * 0.99f) ? mk3(0.0f, 0.5f, 1.0f) : mk3(dbgFrac((1.0f / 100.0f) * sceneLength)); break;
    case kDbgStablePlaneMotionVectors:    c = mk3(0.5f) + mv * mk3(0.2f, 0.2f, 10.0f); break;
    case kDbgStablePlaneNormals:          c = dbgShowNormalSRGB(octUnorm32ToDir(sp.PackedNormal)); break;
    case kDbgStablePlaneRoughness:        c = mk3(f16tof32(sp.VertexIndexAndRoughness & 0xFFFFu)); break;
    case kDbgStablePlaneSpecAvg:          c = mk3(l.w); break;
    case kDbgStablePlaneDiffBSDFEstimate: c = diffEstimate; break;
    case kDbgStablePlaneDiffRadiance:     c = rad * sat(1.0f - l.w / (totalAvg + 1e-12f)); break;
    case kDbgStablePlaneSpecBSDFEstimate: c = specEstimate; break;
    case kDbgStablePlaneSpecRadiance:     c = rad * sat(l.w / (totalAvg + 1e-12f)); break;
    case kDbgStableRadiance:              c = mk3(sqrtf(stableRadiance.x), sqrtf(stableRadiance.y), sqrtf(stableRadiance.z)); break;      // sqrt: RTXPT's "cheap debug tonemapper"
    default: return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    return make_float4(c.x, c.y, c.z, 1.0f);
}

// StablePlanesDebugViz for pixel (px, py) of a W x H image.  P reads the realtime buffers: branchID(x, y, plane), plane(x, y, plane), dominantIndex(x, y), stableRadiance(x, y)
template <class P>
PT_HD float4 stablePlaneDebugPixel(uint view, int dbgPlaneIndex, uint px, uint py, uint W, uint H, const P& buffers)
{
    uint sx = px, sy = py, plane = 0;
    if (view >= kDbgStablePlaneVirtualRayLength && view <= kDbgStablePlaneSpecRadiance) stablePlaneFourWaySplitCoord(dbgPlaneIndex, px, py, W, H, sx, sy, plane);
    const uint branch = plane < 3u ? buffers.branchID(sx, sy, plane) : 0xFFFFFFFFu;
    RtxptStablePlane sp = {};
    if (branch != 0xFFFFFFFFu) sp = buffers.plane(sx, sy, plane);
    return stablePlaneDebugColor(view, px, py, branch, sp, buffers.dominantIndex(px, py), buffers.stableRadiance(px, py));
}

// what DENOISER_FINAL_MERGE's debug switch reads of a pixel (PostProcess.hlsl:596-631): the disocclusion-threshold mix, the denoised radiance after PostDenoiseProcess (both
// zero on sky pixels), view-space depth and the plane's throughput
struct MergeDebugInputs { float relaxedDisocclusion; float3 diff, spec; float viewZ; float3 throughput; };
// one pixel of a merge view (PostProcess.hlsl:658-679).  NRD's validation layer is not part of this library: DenoiserValidation always takes its "validation.a == 0" branch
PT_HD float4 mergeDebugColor(uint view, const MergeDebugInputs& m)
{
    float3 c;
    switch (view)
    {
    case kDbgStablePlaneRelaxedDisocclusion:      return make_float4(sqrtf(m.relaxedDisocclusion), 0.0f, 0.0f, 1.0f);
    case kDbgStablePlaneDiffRadianceDenoised:     c = m.diff; break;
    case kDbgStablePlaneSpecRadianceDenoised:     c = m.spec; break;
    case kDbgStablePlaneViewZ:                    return make_float4(m.viewZ / 10.0f, dbgFrac(m.viewZ), 0.0f, 1.0f);
    case kDbgStablePlaneThroughput:               return make_float4(m.throughput.x, m.throughput.y, m.throughput.z, 1.0f);
    case kDbgStablePlaneCombinedRadianceDenoised:
    case kDbgStablePlaneDenoiserValidation:       c = m.diff + m.spec; break;
    default: return make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    return make_float4(sqrtf(c.x), sqrtf(c.y), sqrtf(c.z), 1.0f);          // sqrt: RTXPT's "cheap debug tonemapper"
}
// where the merge of plane `plane` draws pixel (px, py) (PostProcess.hlsl:637-645): itself, or with the four-way split (-1) into the plane's half-resolution quadrant.  In the
// split, four pixels land on one; RTXPT leaves the winner to the GPU, here the one of even coordinates draws - the pixel StablePlanesDebugViz's split reads for that quadrant.
// Returns false when this pixel draws nothing.  DenoiserValidation draws at the pixel itself (PostProcess.hlsl:671-675)
PT_HD bool mergeDebugTarget(uint view, int dbgPlaneIndex, uint plane, uint px, uint py, uint W, uint H, uint& outX, uint& outY)
{
    outX = px; outY = py;
    if (dbgPlaneIndex >= 0) return uint(dbgPlaneIndex) == plane;
    if (view == kDbgStablePlaneDenoiserValidation) return true;
    if ((px | py) & 1u) return false;
    outX = (plane % 2u) * (W / 2u) + px / 2u; outY = (plane / 2u) * (H / 2u) + py / 2u;
    return true;
}
// the merge of plane 0 with the split fills the quadrants of inactive planes with a checkerboard (PostProcess.hlsl:647-653)
PT_HD bool mergeDebugChecker(int dbgPlaneIndex, uint plane, uint px, uint py, uint W, uint H, uint activePlaneCount)
{
    return dbgPlaneIndex == -1 && plane == 0 && ((px >= W / 2u ? 1u : 0u) + 2u * (py >= H / 2u ? 1u : 0u)) >= activePlaneCount;
}

// the RGBA16F store of DebugPixel (Libraries/ShaderDebug/ShaderDebug.hlsl:637-640)
PT_HD uint2 packDebugPixel(float4 c) { return make_uint2(f32tof16(c.x) | (f32tof16(c.y) << 16), f32tof16(c.z) | (f32tof16(c.w) << 16)); }

} // namespace pt
