// ORACLE — test infrastructure only (see pt_math.h).
// reblur_settings.h: REBLUR_DIFFUSE_SPECULAR under the settings RTXPT's denoiser panel sets (Rtxpt/SampleUI.cpp:1360-1410, m_ui.ReblurSettings, and
// m_ui.NRDUseAlternateDisocclusionThresholdMix), on top of the passes of reblur.h, which restate NRD in RTXPT's default configuration.  What the panel changes beyond reblur.h's
// Settings is gathered in PanelSettings; the frame (denoiseFrameWithSettings) follows NRD's dispatch graph for them (Reblur.cpp:117-160, Reblur_DiffuseSpecular.hpp:83-169):
//   enableHitDistanceReconstruction = hitDistanceReconstructionMode != OFF; skipPrePass = diffusePrepassBlurRadius == 0 && specularPrepassBlurRadius == 0
//   HitDistReconstruction   IN -> ( isPrepassEnabled ? TEMP2 : TEMP1 )                                             (Reblur_DiffuseSpecular.hpp:97-98)
//   PrePass                 ( isAfterReconstruction ? TEMP2 : IN ) -> TEMP1                                        (:117-121)
//   TemporalAccumulation    ( isAfterPrepass ? TEMP1 : IN ), isAfterPrepass = !skipPrePass || enableHitDistanceReconstruction   (:148-149, Reblur.cpp:155)
// AREA_3X3 is REBLUR_DiffuseSpecular_HitDistReconstruction.cs.hlsl: the body of the 5x5 pass (REBLUR_HitDistReconstruction.hlsli:84-98, for j, i in 0 .. 2 * BORDER:
// o = ( i, j ) - BORDER) with BORDER 1 instead of NRD_USE_BORDER_2's 2.
// With specularPrepassBlurRadius 0 TemporalAccumulation takes its tracking hit distance from the specular input and normalises it (REBLUR_TemporalAccumulation.hlsli:32, :125;
// reblur.h temporalAccumulation restates both) - from TEMP1 too at the pixels of its 3x3 that the writing pass skipped (sky tiles, beyond the denoising range), which NRD leaves
// holding whatever an earlier pass wrote there.  Here, as in the library, TEMP1 starts cleared for that case, so that they read as "no hit distance".  A PrePass with one radius 0
// passes that signal through unfiltered (REBLUR_Common_{Diffuse,Specular}SpatialFilter.hlsli:25 / :27; reblur.h spatialPass).  Anti-firefly off skips HistoryFix's 9x9 ring clamp
// (REBLUR_HistoryFix.hlsli:232, :437: gAntiFirefly; reblur.h historyFix's antiFirefly); without the disocclusion-threshold mix (isDisocclusionThresholdMixAvailable false,
// Reblur.cpp:153) TemporalAccumulation reads a mix of 0.  Antilag (gAntilagParams, Reblur.cpp:332) and responsiveAccumulationRoughnessThreshold (:368) reach
// TemporalStabilization / TemporalAccumulation through reblur.h's StabilizationParams / TemporalParams.
#pragma once
#include "reblur.h"

namespace orc { namespace reblur {

struct PanelSettings    // the fields of RtxptReblurSettings (include/rtxpt_b200.h) that reblur.h's Settings does not carry; defaults: RTXPT's
{
    Settings s;
    uint hitDistanceReconstructionMode = 2;                 // 0 OFF, 1 AREA_3X3, 2 AREA_5X5 (NrdConfig.cpp:53)
    bool enableAntiFirefly = true;                          // NrdConfig.cpp:52
    float antilagLuminanceSigmaScale = 4.0f, antilagLuminanceSensitivity = 3.0f;      // nrd::ReblurAntilagSettings
    float responsiveAccumulationRoughnessThreshold = 0.0f;
    bool isDisocclusionThresholdMixAvailable = true;        // SampleUI.h:295
};

// HitDistReconstruction with BORDER 1 (AREA_3X3): reblur.h's hitDistReconstruction line for line with the 3x3 neighbourhood
inline void hitDistReconstruction3x3(const Constants& c, const Inputs& in, const std::vector<uint8_t>& tiles, const Image4& inDiff, const Image4& inSpec, Image4& outDiff, Image4& outSpec)
{
    const int BORDER = 1;
    #pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < int(c.H); y++) for (int x = 0; x < int(c.W); x++)
    {
        if (tileIsSky(c, tiles, x, y)) continue;
        const float viewZ = in.unpackViewZ(x, y, c);
        if (viewZ > c.s.denoisingRange) continue;
        float mid; const float4 nr = in.unpackNormalRoughness(x, y, mid);
        const float3 N = xyz(nr); const float roughness = nr.w;
        const float2 rectSizeInv = f2(1.0f / float(c.W), 1.0f / float(c.H));
        const float2 pixelUv = f2((float(x) + 0.5f) * rectSizeInv.x, (float(y) + 0.5f) * rectSizeInv.y);
        const float3 Xv = ReconstructViewPosition(pixelUv, c, viewZ), Nv = worldToViewRotate(c, N);
        const float frustumSize = GetFrustumSize(c, viewZ);
        const float2 gw = GetGeometryWeightParams(c.s.planeDistanceSensitivity, frustumSize, Xv, Nv), rw = GetRelaxedRoughnessWeightParams(roughness * roughness);
        const float diffNormalW = GetNormalWeightParam(1.0f, 1.0f), specNormalW = GetNormalWeightParam(1.0f, 1.0f, roughness);
        float2 center = f2(inDiff.at(x, y).w, inSpec.at(x, y).w);
        float2 sum = f2(center.x != 0.0f ? 1000.0f : 0.0f, center.y != 0.0f ? 1000.0f : 0.0f);
        center = center * sum;
        for (int j = -BORDER; j <= BORDER; j++) for (int i = -BORDER; i <= BORDER; i++)
        {
            if (i == 0 && j == 0) continue;
            const int sx = std::min(std::max(x + i, 0), int(c.W) - 1), sy = std::min(std::max(y + j, 0), int(c.H) - 1);
            const float2 uv = f2(pixelUv.x + float(i) * rectSizeInv.x, pixelUv.y + float(j) * rectSizeInv.y);
            float w = (uv.x > 0.0f && uv.y > 0.0f && uv.x < 1.0f && uv.y < 1.0f) ? 1.0f : 0.0f;
            w *= GetGaussianWeight(sqrtf(float(i * i + j * j)) * 0.5f);
            const float zs = in.unpackViewZ(sx, sy, c);
            w *= ComputeWeight(dot(Nv, ReconstructViewPosition(uv, c, zs)), gw.x, gw.y);
            float ms; const float4 ns = in.unpackNormalRoughness(sx, sy, ms);
            const float angle = AcosApprox(dot(N, xyz(ns)));
            float2 ww = f2(w * ComputeExponentialWeight(angle, diffNormalW, 0.0f), w * ComputeExponentialWeight(angle, specNormalW, 0.0f) * ComputeExponentialWeight(ns.w * ns.w, rw.x, rw.y));
            float2 data = f2(inDiff.at(sx, sy).w, inSpec.at(sx, sy).w);
            if (ww.x == 0.0f) data.x = 0.0f;
            if (ww.y == 0.0f) data.y = 0.0f;
            ww = f2(data.x != 0.0f ? ww.x : 0.0f, data.y != 0.0f ? ww.y : 0.0f);
            center = center + data * ww; sum = sum + ww;
        }
        center = f2(center.x / std::max(sum.x, NRD_EPS), center.y / std::max(sum.y, NRD_EPS));
        const float4 d = inDiff.at(x, y), s = inSpec.at(x, y);
        outDiff.store(x, y, f4(d.x, d.y, d.z, center.x)); outSpec.store(x, y, f4(s.x, s.y, s.z, center.y));
    }
}

// reblur.h's denoiseFrame with the routing above; with PanelSettings' defaults it runs the passes, images and parameters denoiseFrame does
inline void denoiseFrameWithSettings(const PanelSettings& ps, uint W, uint H, const float* worldToView16, const float* viewToClip16, const float* worldToViewPrev16, const float* viewToClipPrev16,
                                     uint frameIndex, const TemporalParams& tpIn, const Inputs& in, const Image4& inDiff, const Image4& inSpec, History& h, FrameOutputs& out)
{
    const Constants c = makeConstants(ps.s, W, H, worldToView16, viewToClip16, frameIndex);
    if (h.W != W || h.H != H) h.init(W, H);
    TemporalParams tp = tpIn; tp.responsiveAccumulationRoughnessThreshold = ps.responsiveAccumulationRoughnessThreshold;
    if (!ps.isDisocclusionThresholdMixAvailable) tp.disocclusionThresholdMix = nullptr;
    StabilizationParams sp; sp.antilagSigmaScale = ps.antilagLuminanceSigmaScale; sp.antilagSensitivity = ps.antilagLuminanceSensitivity;
    FrameMatrices m;
    memcpy(m.viewToWorld, c.viewToWorld, sizeof(m.viewToWorld));
    auto camPos = [](const float* wv) { return f3(-(wv[12] * wv[0] + wv[13] * wv[1] + wv[14] * wv[2]), -(wv[12] * wv[4] + wv[13] * wv[5] + wv[14] * wv[6]), -(wv[12] * wv[8] + wv[13] * wv[9] + wv[14] * wv[10])); };
    m.cameraDelta = camPos(worldToViewPrev16) - camPos(worldToView16);
    auto relativeWorldToClip = [](const float* wv, float3 camRel, const float* vc, float* outM, float* outAffine) {
        float R[9]; for (int r = 0; r < 3; r++) for (int k = 0; k < 3; k++) R[r * 3 + k] = wv[k * 4 + r];
        const float t[3] = { -(R[0] * camRel.x + R[1] * camRel.y + R[2] * camRel.z), -(R[3] * camRel.x + R[4] * camRel.y + R[5] * camRel.z), -(R[6] * camRel.x + R[7] * camRel.y + R[8] * camRel.z) };
        if (outAffine) for (int r = 0; r < 3; r++) { outAffine[r * 4] = R[r * 3]; outAffine[r * 4 + 1] = R[r * 3 + 1]; outAffine[r * 4 + 2] = R[r * 3 + 2]; outAffine[r * 4 + 3] = t[r]; }
        float wvRel[16] = { R[0], R[3], R[6], 0, R[1], R[4], R[7], 0, R[2], R[5], R[8], 0, t[0], t[1], t[2], 1 };
        for (int r = 0; r < 4; r++) for (int k = 0; k < 4; k++) { float a = 0; for (int j = 0; j < 4; j++) a += wvRel[r * 4 + j] * vc[j * 4 + k]; outM[r * 4 + k] = a; } };
    relativeWorldToClip(worldToView16, f3(0), viewToClip16, m.worldToClip, nullptr);
    relativeWorldToClip(worldToViewPrev16, m.cameraDelta, viewToClipPrev16, m.worldToClipPrev, m.worldToViewPrev);
    { const float P00 = viewToClipPrev16[0], P11 = viewToClipPrev16[5], P20 = viewToClipPrev16[8], P21 = viewToClipPrev16[9]; m.frustumPrev[0] = (-1.0f - P20) / P00; m.frustumPrev[2] = 2.0f / P00; m.frustumPrev[1] = (1.0f - P21) / P11; m.frustumPrev[3] = -2.0f / P11; }
    const size_t n = size_t(W) * H;
    const std::vector<uint8_t> tiles = classifyTiles(c, in);
    Image4 t1d = inDiff, t1s = inSpec, t2d = inDiff, t2s = inSpec;
    auto keep = [&](const Image4& d, const Image4& s) { if (out.keepStages) { out.stageDiff.push_back(d); out.stageSpec.push_back(s); } };
    out.stageDiff.clear(); out.stageSpec.clear();
    const bool reconstruction = ps.hitDistanceReconstructionMode != 0, prePass = c.gDiffPrepassBlurRadius != 0.0f || c.gSpecPrepassBlurRadius != 0.0f;
    if (c.gSpecPrepassBlurRadius == 0.0f && (reconstruction || prePass)) for (float4& v : t1s.v) v = f4(0, 0, 0, 0);
    if (reconstruction)
    {
        Image4& od = prePass ? t2d : t1d; Image4& os = prePass ? t2s : t1s;
        if (ps.hitDistanceReconstructionMode == 1) hitDistReconstruction3x3(c, in, tiles, inDiff, inSpec, od, os);
        else hitDistReconstruction(c, in, tiles, inDiff, inSpec, od, os);
        keep(od, os);
    }
    std::vector<float> prepassTracking(n, 0.0f);
    if (prePass) { SpatialOutputs o{ &t1d, &t1s, &prepassTracking }; spatialPass(c, in, tiles, PRE_BLUR, reconstruction ? t2d : inDiff, reconstruction ? t2s : inSpec, nullptr, o); keep(t1d, t1s); }
    const Image4& taDiff = (reconstruction || prePass) ? t1d : inDiff; const Image4& taSpec = (reconstruction || prePass) ? t1s : inSpec;
    std::vector<float> diffFastT(n, 0.0f), specFastT(n, 0.0f), trackingPong(n, 0.0f);
    out.data1.assign(n * 2, 0); out.data2.assign(n, 0u);
    { TemporalOutputs o{ &t2d, &t2s, &diffFastT, &specFastT, &trackingPong, &out.data1, &out.data2 }; temporalAccumulation(c, m, tp, in, tiles, taDiff, taSpec, prepassTracking, h, o); keep(t2d, t2s); }
    historyFix(c, in, tiles, out.data1, t2d, t2s, diffFastT, specFastT, ps.enableAntiFirefly, 14.0f, h.valid && !tp.resetHistory, t1d, t1s, h.diffFast, h.specFast); keep(t1d, t1s);
    std::vector<float2> frames(n);
    for (size_t i = 0; i < n; i++) frames[i] = f2(float(out.data1[2 * i]) / 255.0f * 63.0f, float(out.data1[2 * i + 1]) / 255.0f * 63.0f);
    { SpatialOutputs o{ &t2d, &t2s, nullptr }; spatialPass(c, in, tiles, BLUR, t1d, t1s, &frames, o); keep(t2d, t2s); }
    for (size_t i = 0; i < n; i++) h.prevViewZ[i] = in.viewZ[i];
    { SpatialOutputs o{ &h.diff, &h.spec, nullptr }; spatialPass(c, in, tiles, POST_BLUR, t2d, t2s, &frames, o); }
    for (size_t i = 0; i < n; i++) h.prevNormalRoughness[i] = in.normalRoughness[i];
    keep(h.diff, h.spec);
    out.diff = h.diff; out.spec = h.spec;
    std::vector<float> lumaD = h.diffLumaStabilized, lumaS = h.specLumaStabilized;
    temporalStabilization(c, m, tp, sp, in, tiles, out.data1, out.data2, h.diff, h.spec, trackingPong, h, out.diff, out.spec, lumaD, lumaS, h.prevInternalData);
    h.diffLumaStabilized.swap(lumaD); h.specLumaStabilized.swap(lumaS); h.specHitDistForTracking.swap(trackingPong);
    h.valid = true;
}

} } // namespace orc::reblur
