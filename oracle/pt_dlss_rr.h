// ORACLE — test infrastructure only (see pt_math.h).  RTXPT's DLSS-RR input pass, PostProcess DLSSRRDenoiserPrepareInputs: the DENOISER_DLSS_RR branch of
// Rtxpt/ProcessingPasses/PostProcess.hlsl:198-411 with ComputeSpecularMotionVector (:94-160), restated over the realtime targets of pt_stable_planes.h.
// MIX_STABLE_RADIANCE, MIX_BY_THROUGHPUT and ALLOW_MIX_NORMALS are 1 (:212-214); primaryLayer feeds only the DenoiserGuide debug views and is not computed.
// Store formats (RenderTargets.cpp:185-197): OutputColor RGBA16F, RRDiffuseAlbedo / RRSpecAlbedo R11G11B10_FLOAT (Pack_R11G11B10_FLOAT: the reference pins no rounding for the
// hardware's store conversion, this is the one the whole library uses), RRNormalsAndRoughness RGBA16F, RRSpecMotionVectors RG16F.
#pragma once
#include "pt_stable_planes.h"

namespace orc {
namespace dlssrr {

// what the pass stores, before the format conversion
struct Result { float3 color, diffAlbedo, specAlbedo, normal; float roughness; float2 specMotion; bool specMotionIsGuide; };

struct View { const float* worldToClip; const float* prevWorldToClip; float clipToWindowScale[2]; };        // matrices row-major, row vector x matrix

inline float4 rowTimes(float3 p, const float* M)        // mul( float4( p, 1 ), M )
{
    float r[4];
    for (int c = 0; c < 4; c++) r[c] = p.x * M[c] + p.y * M[4 + c] + p.z * M[8 + c] + 1.0f * M[12 + c];
    return f4(r[0], r[1], r[2], r[3]);
}

// PostProcess.hlsl:94-160: image of the reflection hit behind a planar reflector (Duff et al. 2017 basis), previous minus current NDC, times clipToWindowScale
inline float2 ComputeSpecularMotionVector(float3 primaryHitPosWorld, float3 primaryRayDirWorld, float3 primaryHitNormalWorld, float3 reflectionRayWorld, const View& v)
{
    float3 principalAxis = primaryHitNormalWorld;
    float zObj = dot(principalAxis, reflectionRayWorld);
    if (zObj < 0.0f) { principalAxis = -principalAxis; zObj = -zObj; }
    zObj = std::max(zObj, 1e-5f);
    const float3 n = principalAxis;
    const float s = n.z < 0.0f ? -1.0f : 1.0f;
    const float a = -1.0f / (s + n.z);
    const float b = n.x * n.y * a;
    const float3 xAxis = f3(1.0f + s * n.x * n.x * a, s * b, -s * n.x);
    const float3 yAxis = f3(b, s + n.y * n.y * a, -n.y);
    const float3 imagePosInReflectorSpace = f3(dot(xAxis, reflectionRayWorld), dot(yAxis, reflectionRayWorld), -zObj);
    const float3 imageInWorld = primaryHitPosWorld + primaryRayDirWorld * length(imagePosInReflectorSpace);
    const float4 prevClip = rowTimes(imageInWorld, v.prevWorldToClip), currClip = rowTimes(imageInWorld, v.worldToClip);
    const float2 prevNdc = f2(prevClip.x / prevClip.w, prevClip.y / prevClip.w), currNdc = f2(currClip.x / currClip.w, currClip.y / currClip.w);
    return f2((prevNdc.x - currNdc.x) * v.clipToWindowScale[0], (prevNdc.y - currNdc.y) * v.clipToWindowScale[1]);
}

inline float3 highHalves(const uint32_t w[3]) { return f3(f16tof32(w[0] >> 16), f16tof32(w[1] >> 16), f16tof32(w[2] >> 16)); }      // UnpackTwoFp32ToFp16's first output
inline float3 lowHalves(const uint32_t w[3]) { return f3(f16tof32(w[0] & 0xFFFF), f16tof32(w[1] & 0xFFFF), f16tof32(w[2] & 0xFFFF)); }

inline Result pixel(const RealtimeTargets& T, const View& v, float brightnessClampK, uint px, uint py)
{
    const size_t pix = size_t(py) * T.width + px;
    const uint dominantStablePlaneIndex = T.LoadDominantIndex(px, py);
    const uint activeCount = T.activePlaneCount();
    Result R;
    float3 combinedRadiance = T.LoadStableRadiance(px, py);
    const float3 stableAlbedo = [&] { const float3 r = ReinhardMax(combinedRadiance); return f3(sqrtf(r.x), sqrtf(r.y), sqrtf(r.z)); }();
    const float stableAlbedoAvg = Average(stableAlbedo);

    float3 guideNormals = f3(0, 0, 1e-6f), diffAlbedo = f3(0), specAlbedo = f3(0);
    float roughness = 0.0f;
    float spWeights[3] = { 0, 0, 0 };
    {
        const float kTW = 0.2f, kNW = 0.01f, kDW = 0.05f;
        float spAvailable[3] = { 1, 0, 0 }, thpWeights[3] = { 1, 0, 0 };
        for (uint i = 1; i < activeCount; i++)
        {
            if (T.GetBranchID(px, py, i) == cStablePlaneInvalidBranchID) continue;
            const float weight = saturate(Average(highHalves(T.planes[T.PixelToAddress(px, py, i)].PackedThpAndMVs)));
            thpWeights[i] = weight;
            thpWeights[0] = saturate(thpWeights[0] - weight);
            spAvailable[i] = 1;
        }
        for (int k = 0; k < 3; k++) spWeights[k] += thpWeights[k] * kTW;
        for (int k = 0; k < 3; k++) spWeights[k] += 1.0f * kNW;
        if (dominantStablePlaneIndex < 3) spWeights[dominantStablePlaneIndex] += kDW;
        for (int k = 0; k < 3; k++) spWeights[k] *= spAvailable[k];
        const float total = spWeights[0] + spWeights[1] + spWeights[2];
        for (int k = 0; k < 3; k++) spWeights[k] /= total;
    }
    for (uint i = 0; i < activeCount; i++)
    {
        if (T.GetBranchID(px, py, i) == cStablePlaneInvalidBranchID) continue;
        const RtxptStablePlane& sp = T.planes[T.PixelToAddress(px, py, i)];
        if (!std::isfinite(sp.SceneLength)) continue;          // sky
        combinedRadiance = combinedRadiance + T.GetNoisyRadiance(sp);
        const float weight = spWeights[i];
        if (weight > 1e-6f)
        {
            guideNormals = guideNormals + f3(weight) * OctToNDirUnorm32(sp.PackedNormal);
            roughness = roughness + weight * f16tof32(sp.VertexIndexAndRoughness & 0xFFFF);
            diffAlbedo = diffAlbedo + f3(weight) * highHalves(sp.DenoiserPackedBSDFEstimate);
            specAlbedo = specAlbedo + f3(weight) * lowHalves(sp.DenoiserPackedBSDFEstimate);
        }
    }
    const float3 stableAlbedoGreyMix = lerp(stableAlbedo, f3(0.5f), 0.2f);
    diffAlbedo = lerp(diffAlbedo, stableAlbedoGreyMix, stableAlbedoAvg / (Average(diffAlbedo) + sqrtf(stableAlbedoAvg) + 1e-7f));
    const float guideNormalsLength = length(guideNormals);
    if (guideNormalsLength < 1e-5f) guideNormals = f3(0, 0, 1); else guideNormals /= guideNormalsLength;
    const float minAlbedo = 0.05f;
    if (Average(diffAlbedo + specAlbedo) < minAlbedo) diffAlbedo = diffAlbedo + f3(minAlbedo);
    const float maxRadiance = max3(combinedRadiance);
    if (maxRadiance > brightnessClampK) combinedRadiance = combinedRadiance * (brightnessClampK / maxRadiance);
    R.color = combinedRadiance; R.diffAlbedo = diffAlbedo; R.specAlbedo = specAlbedo; R.normal = guideNormals; R.roughness = roughness;

    // specular motion vectors (:373-407): plane 0, whether or not it holds a branch
    const RtxptStablePlane& sp = T.planes[T.PixelToAddress(px, py, 0)];
    const float3 rayOrigin = f3(sp.RayOrigin[0], sp.RayOrigin[1], sp.RayOrigin[2]), rayDir = f3(sp.RayDir[0], sp.RayDir[1], sp.RayDir[2]);
    const float3 primaryHitPosWorld = rayOrigin + rayDir * sp.SceneLength;
    const float3 primaryHitNormalWorld = OctToNDirUnorm32(sp.PackedNormal);
    float3 reflectionRayWorld = rayDir - f3(2.0f * dot(primaryHitNormalWorld, rayDir)) * primaryHitNormalWorld;         // reflect()
    const float specHitT = T.specularHitT[pix];
    reflectionRayWorld = reflectionRayWorld * specHitT;
    const float kSpecularRoughnessThreshold = 0.25f;            // PathTracer.hlsli:23
    R.specMotionIsGuide = !(specHitT > 1e-3f && roughness < kSpecularRoughnessThreshold);
    if (R.specMotionIsGuide) R.specMotion = f2(f16tof32(T.motionVectors[pix * 4]), f16tof32(T.motionVectors[pix * 4 + 1]));
    else R.specMotion = ComputeSpecularMotionVector(primaryHitPosWorld, rayDir, primaryHitNormalWorld, reflectionRayWorld, v);
    return R;
}

struct Targets { uint16_t* outputColor; uint32_t* diffAlbedo; uint32_t* specAlbedo; uint16_t* normalsRoughness; uint16_t* specMotion; };     // RGBA16F, R11G11B10 x 2, RGBA16F, RG16F

inline void store(const RealtimeTargets& T, const Targets& O, const Result& R, uint px, uint py)
{
    const size_t pix = size_t(py) * T.width + px;
    storeRGBA16F(O.outputColor + pix * 4, f4(R.color, 1.0f));
    O.diffAlbedo[pix] = Pack_R11G11B10_FLOAT(R.diffAlbedo);
    O.specAlbedo[pix] = Pack_R11G11B10_FLOAT(R.specAlbedo);
    storeRGBA16F(O.normalsRoughness + pix * 4, f4(R.normal, R.roughness));
    if (R.specMotionIsGuide) { O.specMotion[pix * 2] = T.motionVectors[pix * 4]; O.specMotion[pix * 2 + 1] = T.motionVectors[pix * 4 + 1]; }     // the guide's halves as they are
    else { O.specMotion[pix * 2] = uint16_t(f32tof16(R.specMotion.x)); O.specMotion[pix * 2 + 1] = uint16_t(f32tof16(R.specMotion.y)); }
}

} // namespace dlssrr
} // namespace orc
