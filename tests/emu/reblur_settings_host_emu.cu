// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of the product's ReBLUR pass bodies (rtxpt_b200/csrc/reblur_passes.cuh) under the settings of rtxpt_b200_set_reblur_settings: the product's validation, host
// constants and pass routing (reblur_host.h: settingsError, fillFrameParams, routeFrame), run pixel by pixel on the CPU in launchReblurFrame's order.  The settings counterpart of
// reblur_host_emu.cu's rb_emu_denoise (same arguments), so that tests/test_reblur_settings_port.py can hold the routing and the 3x3 reconstruction to the oracle's
// (oracle/reblur_settings.h) without a GPU.
#include "../../rtxpt_b200/csrc/reblur_passes.cuh"
#include "../../rtxpt_b200/csrc/reblur_host.h"
#include <vector>
#include <cstdint>

using namespace pt;

namespace {
struct Instance
{
    uint32_t W = 0, H = 0; bool valid = false; uint32_t pingPong = 0; RtxptReblurSettings settings = rb::defaultSettings();
    std::vector<float> prevViewZ; std::vector<uint32_t> prevNormalRoughness; std::vector<unsigned short> prevInternalData, diffFast, specFast, tracking[2], diffLuma[2], specLuma[2];
    std::vector<uint2> diffHistory, specHistory;
    void init(uint32_t w, uint32_t h)
    {
        W = w; H = h; valid = false; pingPong = 0; const size_t n = size_t(w) * h;
        prevViewZ.assign(n, 0.0f); prevNormalRoughness.assign(n, 0u); prevInternalData.assign(n, 0); diffFast.assign(n, 0); specFast.assign(n, 0); diffHistory.assign(n, make_uint2(0, 0)); specHistory.assign(n, make_uint2(0, 0));
        for (int i = 0; i < 2; i++) { tracking[i].assign(n, 0); diffLuma[i].assign(n, 0); specLuma[i].assign(n, 0); }
    }
};
template <typename F> void forEachPixel(const rb::Params& p, F f)
{
    #pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < int(p.H); y++) for (int x = 0; x < int(p.W); x++) f(x, y);
}
}

extern "C" void* rbs_emu_create() { return new Instance(); }
extern "C" void rbs_emu_destroy(void* p) { delete static_cast<Instance*>(p); }
// rtxpt_b200_set_reblur_settings on this instance: the product's validation, 0 or RTXPT_ERR_INVALID_ARGUMENT (the settings stay)
extern "C" int rbs_emu_set_settings(void* p, const RtxptReblurSettings* s)
{
    if (rb::settingsError(*s)) return RTXPT_ERR_INVALID_ARGUMENT;
    static_cast<Instance*>(p)->settings = *s;
    return 0;
}
// images: RGBA16F as 4 x uint16 per pixel; motion / disocclusionMix may be NULL; outFrames: 2 floats per pixel (accumulated frames after TemporalAccumulation)
extern "C" int rbs_emu_denoise(void* instance, uint32_t W, uint32_t H, const RtxptReblurFrame* frame, const float* viewZ, const uint32_t* normalRoughness, const uint16_t* motion, const uint8_t* disocclusionMix,
                               const uint16_t* inDiff, const uint16_t* inSpec, uint16_t* outDiff, uint16_t* outSpec, float* outFrames)
{
    Instance& h = *static_cast<Instance*>(instance);
    if (h.W != W || h.H != H) h.init(W, H);
    const size_t n = size_t(W) * H, tiles = size_t((W + 15) / 16) * ((H + 15) / 16);
    rb::Params p{}; rb::fillFrameParams(p, W, H, frame, h.valid, h.settings);
    std::vector<unsigned char> tileSky(tiles, 0); std::vector<uint2> tmp1Diff(n, make_uint2(0, 0)), tmp1Spec(n, make_uint2(0, 0)), tmp2Diff(n, make_uint2(0, 0)), tmp2Spec(n, make_uint2(0, 0)), oDiff(n, make_uint2(0, 0)), oSpec(n, make_uint2(0, 0));
    std::vector<unsigned short> trackingT(n, 0), diffFastT(n, 0), specFastT(n, 0); std::vector<uchar2> data1(n, make_uchar2(0, 0)); std::vector<uint32_t> data2(n, 0);
    p.viewZ = viewZ; p.normalRoughness = normalRoughness; p.motion = frame->ignoreMotionVectors ? nullptr : reinterpret_cast<const uint2*>(motion);
    p.disocclusionMix = h.settings.useAlternateDisocclusionThresholdMix ? disocclusionMix : nullptr;          // as rtxpt_b200_reblur_denoise
    p.inDiff = reinterpret_cast<const uint2*>(inDiff); p.inSpec = reinterpret_cast<const uint2*>(inSpec);
    p.tiles = tileSky.data(); p.tmp1Diff = tmp1Diff.data(); p.tmp1Spec = tmp1Spec.data(); p.tmp2Diff = tmp2Diff.data(); p.tmp2Spec = tmp2Spec.data();
    p.trackingTransient = trackingT.data(); p.diffFastTransient = diffFastT.data(); p.specFastTransient = specFastT.data(); p.data1 = data1.data(); p.data2 = data2.data();
    p.prevViewZ = h.prevViewZ.data(); p.prevNormalRoughness = h.prevNormalRoughness.data(); p.prevInternalData = h.prevInternalData.data(); p.diffHistory = h.diffHistory.data(); p.specHistory = h.specHistory.data();
    p.diffFast = h.diffFast.data(); p.specFast = h.specFast.data();
    const uint32_t prev = h.pingPong, curr = prev ^ 1u;
    p.trackingPrev = h.tracking[prev].data(); p.trackingCurr = h.tracking[curr].data(); p.diffLumaPrev = h.diffLuma[prev].data(); p.diffLumaCurr = h.diffLuma[curr].data(); p.specLumaPrev = h.specLuma[prev].data(); p.specLumaCurr = h.specLuma[curr].data();
    p.outDiff = oDiff.data(); p.outSpec = oSpec.data();
    // launchReblurFrame's order and routing
    const rb::FrameRouting r = rb::routeFrame(p, h.settings.hitDistanceReconstructionMode);
    for (uint32_t ty = 0; ty < (H + 15) / 16; ty++) for (uint32_t tx = 0; tx < (W + 15) / 16; tx++)
    {
        int sky = 0;
        for (int j = 0; j < 16; j++) for (int i = 0; i < 16; i++) sky += rb::beyondDenoisingRange(p, int(tx * 16 + i), int(ty * 16 + j)) ? 1 : 0;
        tileSky[size_t(ty) * p.tilesW + tx] = sky == 256 ? 1 : 0;
    }
    if (r.clearSpecTmp1) std::fill(tmp1Spec.begin(), tmp1Spec.end(), make_uint2(0, 0));
    if (r.reconstructionRadius == 2) forEachPixel(p, [&](int x, int y) { rb::hitDistReconstructionPixel<2>(r.reconstruction, x, y); });
    if (r.reconstructionRadius == 1) forEachPixel(p, [&](int x, int y) { rb::hitDistReconstructionPixel<1>(r.reconstruction, x, y); });
    if (r.prePass) forEachPixel(p, [&](int x, int y) { rb::spatialPixel<0>(r.pre, x, y); });
    forEachPixel(p, [&](int x, int y) { rb::temporalAccumulationPixel(r.temporal, x, y); });
    if (outFrames) for (size_t i = 0; i < n; i++) { outFrames[2 * i] = float(data1[i].x) / 255.0f * 63.0f; outFrames[2 * i + 1] = float(data1[i].y) / 255.0f * 63.0f; }
    forEachPixel(p, [&](int x, int y) { rb::historyFixPixel(p, x, y); });
    forEachPixel(p, [&](int x, int y) { rb::spatialPixel<1>(p, x, y); });
    forEachPixel(p, [&](int x, int y) { rb::spatialPixel<2>(p, x, y); });
    forEachPixel(p, [&](int x, int y) { rb::temporalStabilizationPixel(p, x, y); });
    h.pingPong = curr; h.valid = true;
    memcpy(outDiff, oDiff.data(), n * 8); memcpy(outSpec, oSpec.data(), n * 8);
    return 0;
}
