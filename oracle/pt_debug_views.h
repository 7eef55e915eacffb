// ORACLE — test infrastructure only (see pt_math.h).
// RTXPT's debug views restated on the oracle's own types:
//   DbgShowNormalSRGB           PathTracer/PathTracerShared.h:144-147
//   ColorFromHash               PathTracer/Utils/Utils.hlsli:109-112 over Unpack_R11G11B10_FLOAT (Utils/Packing.hlsli:186-192) and Hash32 (Utils/NoiseAndSequences.hlsli:58-69)
//   GradientHeatMap             PathTracer/Utils/Utils.hlsli:92-107
//   StablePlaneDebugVizColor    PathTracer/StablePlanes.hlsli:314-317
//   StablePlaneDebugVizFourWaySplitCoord  PathTracer/StablePlanes.hlsli:321-335
//   surfaceDebugViz             PathTracerBridgeDonut.hlsli:457-510 (the FirstHit_* switch, :490-506)
//   StablePlanesDebugViz        PathTracer/PathTracerDebug.hlsli:359-420 (without the mouse-cursor overlay, :422-455)
//   the DENOISER_FINAL_MERGE views ProcessingPasses/PostProcess.hlsl:596-681
#pragma once
#include "pt_path.h"
#include <cmath>

namespace orc {
namespace dbgviz {

enum : uint
{
    Disabled = 0, DominantStablePlaneIndex = 1, StablePlane_VirtualRayLength = 2, StablePlane_MotionVectors = 3, StablePlane_Normals = 4, StablePlane_Roughness = 5,
    StablePlane_SpecAvg = 6, StablePlane_DiffBSDFEstimate = 7, StablePlane_DiffRadiance = 8, StablePlane_SpecBSDFEstimate = 9, StablePlane_SpecRadiance = 10, StableRadiance = 18,
    FirstHit_Barycentrics = 29, FirstHit_FaceNormal, FirstHit_GeometryNormal, FirstHit_ShadingNormal, FirstHit_ShadingTangent, FirstHit_ShadingBitangent, FirstHit_FrontFacing,
    FirstHit_ThinSurface, FirstHit_Diffuse, FirstHit_Specular, FirstHit_Roughness, FirstHit_Metallic, FirstHit_ShaderID, FirstHit_MaterialID
};

// HLSL leaves pow's precision to the compiler; the oracle takes it in double and rounds once, as the library does, so that the two agree on every fp16 store
inline float Pow22(float x) { return float(std::pow(double(x), double(2.2f))); }
inline float3 DbgShowNormalSRGB(float3 n)
{
    const float3 a = n * 0.5f + f3(0.5f);
    return f3(Pow22(fabsf(a.x)), Pow22(fabsf(a.y)), Pow22(fabsf(a.z)));
}
inline float3 Unpack_R11G11B10_FLOAT(uint rgb) { return f3(f16tof32((rgb << 4) & 0x7FF0), f16tof32((rgb >> 7) & 0x7FF0), f16tof32((rgb >> 17) & 0x7FE0)); }
inline float3 ColorFromHash(uint hash) { return saturate(Unpack_R11G11B10_FLOAT(hash)); }
inline float Smoothstep(float a, float b, float x) { const float t = saturate((x - a) / (b - a)); return t * t * (3.0f - 2.0f * t); }
inline float3 GradientHeatMap(float greyValue)
{
    greyValue = saturate(greyValue);
    float3 heat;
    heat.x = Smoothstep(0.5f, 0.8f, greyValue);
    if (greyValue >= 0.90f) heat.x *= (1.1f - greyValue) * 5.0f;
    heat.y = greyValue > 0.7f ? Smoothstep(1.0f, 0.7f, greyValue) : Smoothstep(0.0f, 0.7f, greyValue);
    heat.z = Smoothstep(1.0f, 0.0f, greyValue);
    if (greyValue <= 0.3f) heat.z *= greyValue / 0.3f;
    return heat;
}
inline float3 StablePlaneDebugVizColor(uint planeIndex) { return f3(float(planeIndex == 0 || planeIndex == 3), float(planeIndex == 1), float(planeIndex == 2 || planeIndex == 3)); }
// returns (x, y, plane)
inline void StablePlaneDebugVizFourWaySplitCoord(int dbgPlaneIndex, uint px, uint py, uint w, uint h, uint out[3])
{
    if (dbgPlaneIndex >= 0) { out[0] = px; out[1] = py; out[2] = uint(dbgPlaneIndex); return; }
    const uint halfX = w / 2, halfY = h / 2, qx = px >= halfX, qy = py >= halfY;
    out[0] = uint((px - qx * halfX) * 2.0); out[1] = uint((py - qy * halfY) * 2.0);
    out[2] = qx + qy * 2;
}

// surfaceDebugViz's switch on the surface Bridge::loadSurface returned; shaderID = 0xFFFFFFFF (no RTXPT_SHADER_ID)
inline float4 SurfaceDebugViz(uint view, const SurfaceData& surface, float2 barycentrics)
{
    const ShadingData& sd = surface.sd; const StandardBSDFData& b = surface.bsdf.data;
    switch (view)
    {
    case FirstHit_Barycentrics:     return f4(barycentrics.x, barycentrics.y, 0.0f, 1.0f);
    case FirstHit_FaceNormal:       { const float3 c = DbgShowNormalSRGB(sd.faceNCorrected); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_GeometryNormal:   { const float3 c = DbgShowNormalSRGB(sd.vertexN); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_ShadingNormal:    { const float3 c = DbgShowNormalSRGB(sd.N); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_ShadingTangent:   { const float3 c = DbgShowNormalSRGB(sd.T); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_ShadingBitangent: { const float3 c = DbgShowNormalSRGB(sd.B); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_FrontFacing:      { const float3 c = saturate(f3(0.15f, 0.1f + float(sd.frontFacing), 0.15f)); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_ThinSurface:      { const float3 c = saturate(f3(0.15f, 0.1f + float(sd.thinSurface), 0.15f)); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_Diffuse:          return f4(b.diffuse.x, b.diffuse.y, b.diffuse.z, 1.0f);
    case FirstHit_Specular:         return f4(b.specular.x, b.specular.y, b.specular.z, 1.0f);
    case FirstHit_Roughness:        return f4(b.roughness, b.roughness, b.roughness, 1.0f);
    case FirstHit_Metallic:         return f4(b.metallic, b.metallic, b.metallic, 1.0f);
    case FirstHit_ShaderID:         { const float3 c = ColorFromHash(Hash32(0xFFFFFFFFu)); return f4(c.x, c.y, c.z, 1.0f); }
    case FirstHit_MaterialID:       { const float3 c = ColorFromHash(Hash32(sd.materialID)); return f4(c.x, c.y, c.z, 1.0f); }
    default:                        return f4(0, 0, 0, 0);
    }
}

// StablePlanesDebugViz for one pixel; alpha 0 = nothing drawn
inline float4 StablePlanesDebugViz(const RealtimeTargets& T, uint view, int dbgPlaneIndex, uint px, uint py)
{
    if ((view == Disabled || view > StablePlane_SpecRadiance) && view != StableRadiance) return f4(0, 0, 0, 0);
    uint displayPos[3] = { px, py, 0 };
    if (view >= StablePlane_VirtualRayLength && view <= StablePlane_SpecRadiance) StablePlaneDebugVizFourWaySplitCoord(dbgPlaneIndex, px, py, T.width, T.height, displayPos);
    uint stableBranchID = cStablePlaneInvalidBranchID;
    if (displayPos[2] < cStablePlaneCount) stableBranchID = T.GetBranchID(displayPos[0], displayPos[1], displayPos[2]);
    if (stableBranchID == cStablePlaneInvalidBranchID) { const float c = float((px + py) % 2); return f4(c, c, c, 1.0f); }
    const RtxptStablePlane& sp = T.planes[T.PixelToAddress(displayPos[0], displayPos[1], displayPos[2])];
    const float sceneLength = sp.SceneLength;
    float3 thp, motionVectors; UnpackTwoFp32ToFp16(sp.PackedThpAndMVs, thp, motionVectors);
    float3 diffBSDFEstimate, specBSDFEstimate; UnpackTwoFp32ToFp16(sp.DenoiserPackedBSDFEstimate, diffBSDFEstimate, specBSDFEstimate);
    const float rangeVizScale = 1.0f / 100.0f;
    const float3 sceneLengthCol = (sceneLength >= kMaxRayTravel * 0.99f) ? f3(0, 0.5f, 1) : f3(rangeVizScale * sceneLength - floorf(rangeVizScale * sceneLength));
    const float2 a = Fp16ToFp32(sp.PackedNoisyRadianceAndSpecAvg[0]), b = Fp16ToFp32(sp.PackedNoisyRadianceAndSpecAvg[1]);
    const float4 l = f4(a.x, a.y, b.x, b.y);
    const float3 rad = f3(l.x, l.y, l.z);
    const float totalAvg = Average(rad);
    const float3 diff = rad * saturate(1.0f - (l.w * 1.0f) / (totalAvg + 1e-12f));
    const float3 spec = rad * saturate((l.w * 1.0f) / (totalAvg + 1e-12f));
    const uint dominantSP = T.LoadDominantIndex(px, py);
    float3 c;
    switch (view)
    {
    case DominantStablePlaneIndex:      c = StablePlaneDebugVizColor(dominantSP); break;
    case StablePlane_VirtualRayLength:  c = sceneLengthCol; break;
    case StablePlane_MotionVectors:     c = f3(0.5f) + motionVectors * f3(0.2f, 0.2f, 10.0f); break;
    case StablePlane_Normals:           c = DbgShowNormalSRGB(OctToNDirUnorm32(sp.PackedNormal)); break;
    case StablePlane_Roughness:         c = f3(f16tof32(sp.VertexIndexAndRoughness & 0xFFFF)); break;
    case StablePlane_SpecAvg:           c = f3(l.w); break;
    case StablePlane_DiffBSDFEstimate:  c = diffBSDFEstimate; break;
    case StablePlane_DiffRadiance:      c = diff; break;
    case StablePlane_SpecBSDFEstimate:  c = specBSDFEstimate; break;
    case StablePlane_SpecRadiance:      c = spec; break;
    default:                            { const float3 s = T.LoadStableRadiance(px, py); c = f3(sqrtf(s.x), sqrtf(s.y), sqrtf(s.z)); break; }     // StableRadiance
    }
    return f4(c.x, c.y, c.z, 1.0f);
}

// DENOISER_FINAL_MERGE of plane `stablePlaneIndex` with its debug views: every pixel in turn, drawing into `viz` (RGBA32F, full image) as DebugPixel would.  Where four pixels
// land on one quadrant pixel of the split (dbgPlaneIndex -1), RTXPT leaves the winner to the GPU; the pixel of even coordinates draws, the one StablePlanesDebugViz's split reads.
// NRD's validation layer is absent: t_DenoiserValidation reads 0
enum : uint { StablePlane_RelaxedDisocclusion = 11, StablePlane_DiffRadianceDenoised, StablePlane_SpecRadianceDenoised, StablePlane_CombinedRadianceDenoised, StablePlane_ViewZ,
              StablePlane_Throughput, StablePlane_DenoiserValidation };
inline void DenoiserFinalMergeDebugViz(const RealtimeTargets& T, const DenoiserTargets& D, uint stablePlaneIndex, int dbgPlaneIndex, uint view, const uint16_t* denoisedDiff,
                                       const uint16_t* denoisedSpec, float* viz)
{
    if (view < StablePlane_RelaxedDisocclusion || view > StablePlane_DenoiserValidation) return;
    auto DebugPixel = [&](uint x, uint y, float4 c) { float* o = viz + (size_t(y) * T.width + x) * 4; o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = c.w; };
    for (uint py = 0; py < T.height; py++)
        for (uint px = 0; px < T.width; px++)
        {
            const size_t pix = size_t(py) * T.width + px;
            float3 diffRadiance = f3(0), specRadiance = f3(0); float relaxedDisocclusion = 0;
            const bool hasSurface = D.viewZ[pix] != 3.402823466e+38f;
            const RtxptStablePlane& sp = T.planes[T.PixelToAddress(px, py, stablePlaneIndex)];
            if (hasSurface)
            {
                float3 diffBSDFEstimate, specBSDFEstimate; UnpackTwoFp32ToFp16(sp.DenoiserPackedBSDFEstimate, diffBSDFEstimate, specBSDFEstimate);
                relaxedDisocclusion = float(D.disocclusionMix[pix]) / 255.0f;
                auto load = [&](const uint16_t* p) { return f3(f16tof32(p[pix * 4]), f16tof32(p[pix * 4 + 1]), f16tof32(p[pix * 4 + 2])); };
                diffRadiance = NRD_YCoCgToLinear(load(denoisedDiff)) * diffBSDFEstimate;      // DenoiserNRD::PostDenoiseProcess
                specRadiance = NRD_YCoCgToLinear(load(denoisedSpec)) * specBSDFEstimate;
            }
            bool debugThisPlane = dbgPlaneIndex == int(stablePlaneIndex);
            uint outX = px, outY = py;
            const uint halfX = T.width / 2, halfY = T.height / 2;
            if (dbgPlaneIndex == -1)
            {
                debugThisPlane = (px % 2 == 0) && (py % 2 == 0);
                outX = (stablePlaneIndex % 2) * halfX + px / 2; outY = (stablePlaneIndex / 2) * halfY + py / 2;
            }
            if (dbgPlaneIndex == -1 && stablePlaneIndex == 0)
            {
                const uint quadPlaneIndex = uint(px >= halfX) + 2 * uint(py >= halfY);
                if (quadPlaneIndex >= T.rt->activeStablePlaneCount) { const float c = float((px + py) % 2); DebugPixel(px, py, f4(c, c, c, 1)); }
            }
            if (view == StablePlane_DenoiserValidation && dbgPlaneIndex == -1) debugThisPlane = true;        // drawn at the pixel itself
            if (!debugThisPlane) continue;
            const float viewZ = D.viewZ[pix];
            float3 throughput, motionVectors; UnpackTwoFp32ToFp16(sp.PackedThpAndMVs, throughput, motionVectors);
            const float3 comb = diffRadiance + specRadiance;
            switch (view)
            {
            case StablePlane_RelaxedDisocclusion:      DebugPixel(outX, outY, f4(sqrtf(relaxedDisocclusion), 0, 0, 1)); break;
            case StablePlane_DiffRadianceDenoised:     DebugPixel(outX, outY, f4(sqrtf(diffRadiance.x), sqrtf(diffRadiance.y), sqrtf(diffRadiance.z), 1)); break;
            case StablePlane_SpecRadianceDenoised:     DebugPixel(outX, outY, f4(sqrtf(specRadiance.x), sqrtf(specRadiance.y), sqrtf(specRadiance.z), 1)); break;
            case StablePlane_CombinedRadianceDenoised: DebugPixel(outX, outY, f4(sqrtf(comb.x), sqrtf(comb.y), sqrtf(comb.z), 1)); break;
            case StablePlane_ViewZ:                    DebugPixel(outX, outY, f4(viewZ / 10, viewZ - floorf(viewZ), 0, 1)); break;
            case StablePlane_Throughput:               DebugPixel(outX, outY, f4(throughput.x, throughput.y, throughput.z, 1)); break;
            default:                                   DebugPixel(px, py, f4(sqrtf(comb.x), sqrtf(comb.y), sqrtf(comb.z), 1)); break;       // validation.a == 0
            }
        }
}

} // namespace dbgviz
} // namespace orc
