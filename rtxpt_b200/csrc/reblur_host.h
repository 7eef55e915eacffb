// reblur_host.h - host half of the ReBLUR denoiser: nrd::ReblurSettings (RTXPT's defaults: Rtxpt/NRD/NrdConfig.cpp:49-61; the fields its panel sets: RtxptReblurSettings), nrd::CommonSettings (NrdIntegration.cpp:375-408) and the
// per-frame constants NRD derives from the matrices (External/Nrd/Source/InstanceImpl.cpp:331-451, Reblur.cpp:280-392): camera-relative matrices, frustum, unproject, kernel
// rotators, and the pass routing the settings select.  Plain C++ on top of rb::Params; used by api.cu, reblur_kernels.cu and by the test-only host builds of the passes (tests/emu/reblur_host_emu.cu, reblur_settings_host_emu.cu).
#pragma once
#include "reblur.cuh"
#include "../../include/rtxpt_b200.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace pt { namespace rb {

inline Rotator rbRotator(float angle) { const float ca = cosf(angle), sa = sinf(angle); return { ca, sa, -sa, ca }; }
inline Rotator rbCombine(Rotator a, Rotator b) { return { a.x * b.x + a.z * b.y, a.y * b.x + a.w * b.y, a.x * b.z + a.z * b.w, a.y * b.z + a.w * b.w }; }
inline float rbWeyl(float p, uint32_t n) { const float v = p + float(n) * 0.6180339887498948f; return v - floorf(v); }
inline void rbFrustum(const float* viewToClip, float* f) { const float P00 = viewToClip[0], P11 = viewToClip[5], P20 = viewToClip[8], P21 = viewToClip[9]; f[0] = (-1.0f - P20) / P00; f[2] = 2.0f / P00; f[1] = (1.0f - P21) / P11; f[3] = -2.0f / P11; }
inline void rbCameraPosition(const float* wv, float* o) { for (int k = 0; k < 3; k++) o[k] = -(wv[12] * wv[k * 4] + wv[13] * wv[k * 4 + 1] + wv[14] * wv[k * 4 + 2]); }
// world (relative to the current camera) -> clip of the camera that sits at camRel; optionally the 3x4 world -> view of that camera
inline void rbRelativeWorldToClip(const float* wv, const float* camRel, const float* vc, float* outM, float* outAffine)
{
    float R[9]; for (int r = 0; r < 3; r++) for (int k = 0; k < 3; k++) R[r * 3 + k] = wv[k * 4 + r];
    const float t[3] = { -(R[0] * camRel[0] + R[1] * camRel[1] + R[2] * camRel[2]), -(R[3] * camRel[0] + R[4] * camRel[1] + R[5] * camRel[2]), -(R[6] * camRel[0] + R[7] * camRel[1] + R[8] * camRel[2]) };
    if (outAffine) for (int r = 0; r < 3; r++) { outAffine[r * 4] = R[r * 3]; outAffine[r * 4 + 1] = R[r * 3 + 1]; outAffine[r * 4 + 2] = R[r * 3 + 2]; outAffine[r * 4 + 3] = t[r]; }
    const float wvRel[16] = { R[0], R[3], R[6], 0, R[1], R[4], R[7], 0, R[2], R[5], R[8], 0, t[0], t[1], t[2], 1 };
    for (int r = 0; r < 4; r++) for (int k = 0; k < 4; k++) { float a = 0; for (int j = 0; j < 4; j++) a += wvRel[r * 4 + j] * vc[j * 4 + k]; outM[r * 4 + k] = a; }
}


// nrd::ReblurSettings defaults (NRDSettings.h:230-300) with RTXPT's overrides (Rtxpt/NRD/NrdConfig.cpp:49-61): enableAntiFirefly, AREA_5X5, maxAccumulatedFrameNum 50, pre-pass radii 15 / 40
inline RtxptReblurSettings defaultSettings()
{
    RtxptReblurSettings s;
    s.hitDistanceParameters[0] = 3.0f; s.hitDistanceParameters[1] = 0.1f; s.hitDistanceParameters[2] = 20.0f; s.hitDistanceParameters[3] = -25.0f;
    s.antilagLuminanceSigmaScale = 4.0f; s.antilagLuminanceSensitivity = 3.0f;
    s.maxAccumulatedFrameNum = 50; s.maxFastAccumulatedFrameNum = 6; s.historyFixFrameNum = 3;
    s.diffusePrepassBlurRadius = 15.0f; s.specularPrepassBlurRadius = 40.0f; s.minBlurRadius = 1.0f; s.maxBlurRadius = 30.0f;
    s.lobeAngleFraction = 0.15f; s.roughnessFraction = 0.15f; s.responsiveAccumulationRoughnessThreshold = 0.0f; s.planeDistanceSensitivity = 0.02f;
    s.hitDistanceReconstructionMode = RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5; s.enableAntiFirefly = 1; s.useAlternateDisocclusionThresholdMix = 1;
    return s;
}
// what rtxpt_b200_set_reblur_settings refuses: NULL when `s` is accepted, else the reason
inline const char* settingsError(const RtxptReblurSettings& s)
{
    const float all[] = { s.hitDistanceParameters[0], s.hitDistanceParameters[1], s.hitDistanceParameters[2], s.hitDistanceParameters[3], s.antilagLuminanceSigmaScale, s.antilagLuminanceSensitivity,
                          s.diffusePrepassBlurRadius, s.specularPrepassBlurRadius, s.minBlurRadius, s.maxBlurRadius, s.lobeAngleFraction, s.roughnessFraction,
                          s.responsiveAccumulationRoughnessThreshold, s.planeDistanceSensitivity };
    for (float v : all) if (!std::isfinite(v)) return "every value must be finite";
    if (s.diffusePrepassBlurRadius < 0.0f || s.specularPrepassBlurRadius < 0.0f || s.minBlurRadius < 0.0f || s.maxBlurRadius < 0.0f) return "radii must not be negative";
    const float fractions[] = { s.lobeAngleFraction, s.roughnessFraction, s.responsiveAccumulationRoughnessThreshold, s.planeDistanceSensitivity };
    for (float v : fractions) if (v < 0.0f || v > 1.0f) return "lobeAngleFraction, roughnessFraction, responsiveAccumulationRoughnessThreshold and planeDistanceSensitivity lie in [0, 1]";
    if (s.maxAccumulatedFrameNum > 63 || s.maxFastAccumulatedFrameNum > 63 || s.historyFixFrameNum > 63) return "frame counts lie in [0, 63] (REBLUR_MAX_HISTORY_FRAME_NUM)";
    if (s.hitDistanceReconstructionMode > RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5) return "hitDistanceReconstructionMode: OFF (0), AREA_3X3 (1) or AREA_5X5 (2)";
    if (s.enableAntiFirefly > 1 || s.useAlternateDisocclusionThresholdMix > 1) return "enableAntiFirefly and useAlternateDisocclusionThresholdMix are 0 or 1";
    return nullptr;
}

// everything of rb::Params except the resource pointers, for settings `s`; historyValid = this plane's instance has denoised a frame since its creation / last resize
inline void fillFrameParams(Params& p, uint32_t W, uint32_t H, const RtxptReblurFrame* f, bool historyValid, const RtxptReblurSettings& s = defaultSettings())
{
    p.W = W; p.H = H; p.tilesW = (W + 15) / 16; p.frameIndex = f->frameIndex;
    for (int r = 0; r < 3; r++) for (int k = 0; k < 3; k++) p.viewToWorld[r * 3 + k] = f->matWorldToView[k * 4 + r];
    memcpy(p.viewToClip, f->matViewToClip, 64);
    rbFrustum(f->matViewToClip, p.frustum); rbFrustum(f->prevMatViewToClip, p.frustumPrev);
    float pos[3], posPrev[3]; rbCameraPosition(f->matWorldToView, pos); rbCameraPosition(f->prevMatWorldToView, posPrev);
    for (int k = 0; k < 3; k++) p.cameraDelta[k] = posPrev[k] - pos[k];
    const float zero[3] = { 0, 0, 0 };
    rbRelativeWorldToClip(f->matWorldToView, zero, f->matViewToClip, p.worldToClip, nullptr);
    rbRelativeWorldToClip(f->prevMatWorldToView, p.cameraDelta, f->prevMatViewToClip, p.worldToClipPrev, p.worldToViewPrev);
    p.unproject = 1.0f / (0.5f * float(H) * f->matViewToClip[5]); p.minRectDimMulUnproject = float(std::min(W, H)) * p.unproject;
    const float rad90 = 1.5707963267948966f, rad360 = 6.283185307179586f;
    p.rotatorPre = rbRotator(rbWeyl(0.5f, f->frameIndex) * rad90);
    p.rotator = rbCombine(rbRotator(rbWeyl(0.0f, f->frameIndex * 2) * rad90), rbRotator(float((f->frameIndex * 2) & 15u) / 16.0f * rad360));
    p.rotatorPost = rbCombine(rbRotator(rbWeyl(0.0f, f->frameIndex * 2 + 1) * rad90), rbRotator(float((f->frameIndex * 2 + 1) & 15u) / 16.0f * rad360));
    // settings (AddSharedConstants_Reblur, Reblur.cpp:284-388); the rest are NRD's defaults, which RTXPT's panel does not expose
    const bool reset = f->resetHistory != 0 || !historyValid;
    memcpy(p.hitDistParams, s.hitDistanceParameters, 16);
    p.maxAccumulatedFrameNum = reset ? 0.0f : float(std::min(s.maxAccumulatedFrameNum, 63u)); p.maxFastAccumulatedFrameNum = reset ? 0.0f : float(s.maxFastAccumulatedFrameNum);
    p.historyFixFrameNum = float(s.historyFixFrameNum); p.historyFixBasePixelStride = 14.0f;
    p.diffPrepassBlurRadius = s.diffusePrepassBlurRadius; p.specPrepassBlurRadius = s.specularPrepassBlurRadius; p.minBlurRadius = s.minBlurRadius; p.maxBlurRadius = std::max(s.maxBlurRadius, s.minBlurRadius);
    p.lobeAngleFraction = s.lobeAngleFraction * s.lobeAngleFraction; p.roughnessFraction = s.roughnessFraction;
    p.planeDistSensitivity = s.planeDistanceSensitivity; p.minHitDistanceWeight = 0.1f; p.minMaterialDiff = 4.0f; p.minMaterialSpec = 4.0f; p.denoisingRange = 100000.0f; p.viewZScale = 1.0f;
    const float thresholdBonus = 1.0f / float(H);           // ( 1 + jitterDelta ) / rectH, Reblur.cpp:293; un-jittered matrices
    p.disocclusionThreshold = (f->disocclusionThreshold > 0.0f ? f->disocclusionThreshold : 0.03f) + thresholdBonus;
    p.disocclusionThresholdAlternate = (f->disocclusionThresholdAlternate > 0.0f ? f->disocclusionThresholdAlternate : 0.2f) + thresholdBonus;
    p.framerateScale = f->frameTimeMs > 0.0f ? std::max(33.333f / f->frameTimeMs, 1.0f) : 2.0f;          // max( 33.333 ms / frame time, 1 ), Reblur.cpp:296
    p.fireflySuppressorMinRelativeScale = 2.0f; p.responsiveAccumulationRoughnessThreshold = s.responsiveAccumulationRoughnessThreshold;
    p.antilagSigmaScale = s.antilagLuminanceSigmaScale; p.antilagSensitivity = s.antilagLuminanceSensitivity; p.stabilizationStrength = reset ? 0.0f : 63.0f / 64.0f;
    p.antiFirefly = s.enableAntiFirefly; p.usePrepassOnlyForSpecularMotionEstimation = 0;
}

// NRD's dispatch graph for the settings (Reblur.cpp:117-160, Reblur_DiffuseSpecular.hpp:83-169): which of HitDistReconstruction and PrePass run, and the Params each pass of
// the three at the head of the chain is launched with.  The pass bodies read and write fixed fields (reconstruction: in -> tmp2, PrePass: tmp2 -> tmp1, TemporalAccumulation:
// tmp1 -> tmp2); the routing points those fields at the images NRD binds for the permutation:
//   HitDistReconstruction   -> TEMP2 ahead of a PrePass, else -> TEMP1
//   PrePass                 TEMP2 after a reconstruction, else IN ->
//   TemporalAccumulation    TEMP1 after either of them, else IN
// clearSpecTmp1: TemporalAccumulation reads the hit distance of its 3x3 neighbourhood from its specular input when specularPrepassBlurRadius is 0 (REBLUR_TemporalAccumulation.hlsli:32);
// when that input is TEMP1, the pixels the writing pass skips (sky tiles, beyond the denoising range) would hold whatever an earlier pass left there, which NRD leaves undefined.
// TEMP1 is cleared first, so that they read as "no hit distance".
struct FrameRouting { int reconstructionRadius; bool prePass, clearSpecTmp1; Params reconstruction, pre, temporal; };
inline FrameRouting routeFrame(const Params& p, uint32_t hitDistanceReconstructionMode)
{
    FrameRouting r;
    r.reconstructionRadius = hitDistanceReconstructionMode == RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5 ? 2 : (hitDistanceReconstructionMode == RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_3X3 ? 1 : 0);
    r.prePass = p.diffPrepassBlurRadius != 0.0f || p.specPrepassBlurRadius != 0.0f;
    r.clearSpecTmp1 = p.specPrepassBlurRadius == 0.0f && (r.reconstructionRadius != 0 || r.prePass);
    r.reconstruction = p; r.pre = p; r.temporal = p;
    if (!r.prePass) { r.reconstruction.tmp2Diff = p.tmp1Diff; r.reconstruction.tmp2Spec = p.tmp1Spec; }
    if (r.reconstructionRadius == 0) { r.pre.tmp2Diff = const_cast<uint2*>(p.inDiff); r.pre.tmp2Spec = const_cast<uint2*>(p.inSpec); }
    if (r.reconstructionRadius == 0 && !r.prePass) { r.temporal.tmp1Diff = const_cast<uint2*>(p.inDiff); r.temporal.tmp1Spec = const_cast<uint2*>(p.inSpec); }
    return r;
}

} } // namespace pt::rb
