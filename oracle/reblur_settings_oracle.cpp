// ORACLE build with ReBLUR's panel settings — test infrastructure only.  The committed oracle (oracle.cpp, unchanged) plus one ReBLUR instance kind that carries settings
// (reblur_settings.h): oracle_reblur_settings_create / _destroy / _set / _denoise.  _denoise takes the arguments of oracle_reblur_denoise.
#include "oracle.cpp"
#include "reblur_settings.h"

struct ReblurSettingsInstance { orc::reblur::History history; orc::reblur::FrameOutputs last; orc::reblur::PanelSettings settings; };      // settings: RTXPT's until _set

extern "C" {

ORC_API void* oracle_reblur_settings_create() { return new ReblurSettingsInstance(); }
ORC_API void oracle_reblur_settings_destroy(void* p) { delete (ReblurSettingsInstance*)p; }
// nrd::SetDenoiserSettings with the fields of RtxptReblurSettings (include/rtxpt_b200.h) for the instance's next frames; the history stays.  No validation: the caller passes
// settings the library accepts.
ORC_API int oracle_reblur_settings_set(void* p, const RtxptReblurSettings* u)
{
    if (!p || !u) return -1;
    orc::reblur::PanelSettings& ps = ((ReblurSettingsInstance*)p)->settings; orc::reblur::Settings& s = ps.s;
    memcpy(s.hitDistParams, u->hitDistanceParameters, 16);
    s.maxAccumulatedFrameNum = u->maxAccumulatedFrameNum; s.maxFastAccumulatedFrameNum = u->maxFastAccumulatedFrameNum; s.historyFixFrameNum = u->historyFixFrameNum;
    s.diffusePrepassBlurRadius = u->diffusePrepassBlurRadius; s.specularPrepassBlurRadius = u->specularPrepassBlurRadius; s.minBlurRadius = u->minBlurRadius; s.maxBlurRadius = u->maxBlurRadius;
    s.lobeAngleFraction = u->lobeAngleFraction; s.roughnessFraction = u->roughnessFraction; s.planeDistanceSensitivity = u->planeDistanceSensitivity;
    ps.antilagLuminanceSigmaScale = u->antilagLuminanceSigmaScale; ps.antilagLuminanceSensitivity = u->antilagLuminanceSensitivity;
    ps.responsiveAccumulationRoughnessThreshold = u->responsiveAccumulationRoughnessThreshold; ps.hitDistanceReconstructionMode = u->hitDistanceReconstructionMode;
    ps.enableAntiFirefly = u->enableAntiFirefly != 0; ps.isDisocclusionThresholdMixAvailable = u->useAlternateDisocclusionThresholdMix != 0;
    return 0;
}
ORC_API int oracle_reblur_settings_denoise(void* p, uint32_t W, uint32_t H, const float* worldToView16, const float* viewToClip16, const float* worldToViewPrev16, const float* viewToClipPrev16,
                                           uint32_t frameIndex, int resetHistory, const float* viewZ, const uint32_t* normalRoughness, const uint16_t* motion, const uint8_t* disocclusionMix,
                                           const uint16_t* inDiff, const uint16_t* inSpec, uint16_t* outDiff, uint16_t* outSpec, float* outAccumFrames)
{
    using namespace orc::reblur;
    ReblurSettingsInstance* inst = (ReblurSettingsInstance*)p;
    Inputs in; in.W = W; in.H = H; in.viewZ = viewZ; in.normalRoughness = normalRoughness;
    TemporalParams tp; tp.motion = motion; tp.disocclusionThresholdMix = disocclusionMix; tp.resetHistory = resetHistory != 0;
    tp.disocclusionThreshold = 0.03f + 1.0f / float(H); tp.disocclusionThresholdAlternate = 0.2f + 1.0f / float(H);      // as oracle_reblur_denoise
    const size_t n = size_t(W) * H;
    Image4 d, s; d.init(W, H); s.init(W, H);
    for (size_t i = 0; i < n; i++) { d.v[i] = f4(f16tof32(inDiff[4 * i]), f16tof32(inDiff[4 * i + 1]), f16tof32(inDiff[4 * i + 2]), f16tof32(inDiff[4 * i + 3])); s.v[i] = f4(f16tof32(inSpec[4 * i]), f16tof32(inSpec[4 * i + 1]), f16tof32(inSpec[4 * i + 2]), f16tof32(inSpec[4 * i + 3])); }
    denoiseFrameWithSettings(inst->settings, W, H, worldToView16, viewToClip16, worldToViewPrev16, viewToClipPrev16, frameIndex, tp, in, d, s, inst->history, inst->last);
    for (size_t i = 0; i < n; i++)
    {
        const float4 a = inst->last.diff.v[i], b = inst->last.spec.v[i];
        outDiff[4 * i] = uint16_t(f32tof16(a.x)); outDiff[4 * i + 1] = uint16_t(f32tof16(a.y)); outDiff[4 * i + 2] = uint16_t(f32tof16(a.z)); outDiff[4 * i + 3] = uint16_t(f32tof16(a.w));
        outSpec[4 * i] = uint16_t(f32tof16(b.x)); outSpec[4 * i + 1] = uint16_t(f32tof16(b.y)); outSpec[4 * i + 2] = uint16_t(f32tof16(b.z)); outSpec[4 * i + 3] = uint16_t(f32tof16(b.w));
        if (outAccumFrames) { outAccumFrames[2 * i] = float(inst->last.data1[2 * i]) / 255.0f * 63.0f; outAccumFrames[2 * i + 1] = float(inst->last.data1[2 * i + 1]) / 255.0f * 63.0f; }
    }
    return 0;
}

} // extern "C"
