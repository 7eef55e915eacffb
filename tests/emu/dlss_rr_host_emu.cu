// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of the DLSS-RR input pass (rtxpt_b200/csrc/denoiser_iface.cuh: dlssRrPixel / dnPrepareDlssRrPixel, the bodies k_dn_prepare_dlss_rr runs) for
// tests/test_dlss_rr_port.py, which holds it to the reference's known answers (tests/golden/dlss_rr_golden.npz) and to the oracle's restatement (oracle/pt_dlss_rr.h).  Built by
// dlss_rr.mk.
#include "../../rtxpt_b200/csrc/denoiser_iface.cuh"
#include <cstring>

using namespace pt;

namespace {
LaunchParams frameParams(uint32_t W, uint32_t H, const RtxptRealtimeConstants* rt, RtxptStablePlane* planes, uint32_t* header, uint2* stableRadiance, uint2* motion, float* specHitT)
{
    LaunchParams p; memset(&p, 0, sizeof(p));
    p.c.imageWidth = W; p.c.imageHeight = H;
    p.rt.planes = planes; p.rt.header = header; p.rt.stableRadiance = stableRadiance; p.rt.specularHitT = specHitT; p.motionVectors = motion;
    p.rt.lineStride = ((W + 7u) / 8u) * 8u; p.rt.planeStride = p.rt.lineStride * ((H + 7u) / 8u) * 8u;
    p.rt.activePlaneCount = rt->activeStablePlaneCount;
    memcpy(p.rt.worldToClipNoOffset, rt->matWorldToClipNoOffset, 64); memcpy(p.rt.prevWorldToClipNoOffset, rt->prevMatWorldToClipNoOffset, 64);
    p.rt.clipToWindowScale[0] = rt->clipToWindowScale[0]; p.rt.clipToWindowScale[1] = rt->clipToWindowScale[1];
    return p;
}
}

// records of ref_kat_dlss_rr (104 words) -> 15 floats each: what the pass computes before the stores
extern "C" void dlss_rr_emu_records(const uint32_t* in, uint32_t count, float* out)
{
    RtxptStablePlane planes[3 * 64]; uint32_t header[4]; uint2 stableRadiance, motion; float specHitT;
    for (uint32_t i = 0; i < count; i++, in += 104, out += 15)
    {
        RtxptRealtimeConstants rt{}; rt.activeStablePlaneCount = in[0];
        memcpy(rt.matWorldToClipNoOffset, in + 70, 64); memcpy(rt.prevMatWorldToClipNoOffset, in + 86, 64); memcpy(rt.clipToWindowScale, in + 102, 8);
        LaunchParams p = frameParams(1, 1, &rt, planes, header, &stableRadiance, &motion, &specHitT);
        memcpy(header, in + 2, 16);
        memset(planes, 0, sizeof(planes));
        for (uint k = 0; k < 3; k++) memcpy(&planes[planeAddress(p.rt, 0, k)], in + 6 + 20 * k, 80);
        stableRadiance = make_uint2(in[66], in[67]); memcpy(&specHitT, in + 68, 4); motion = make_uint2(in[69], 0u);
        float clampK; memcpy(&clampK, in + 1, 4);
        const DlssRrPixel r = dlssRrPixel(p, 0u, clampK);
        const float o[15] = { r.color.x, r.color.y, r.color.z, r.diffAlbedo.x, r.diffAlbedo.y, r.diffAlbedo.z, r.specAlbedo.x, r.specAlbedo.y, r.specAlbedo.z,
                              r.normal.x, r.normal.y, r.normal.z, r.roughness, r.specMotion.x, r.specMotion.y };
        memcpy(out, o, sizeof(o));
    }
}

// the pass over a whole frame, in the targets' formats (the arguments of oracle_dlss_rr_frame): planes, header, stable radiance and motion vectors (RGBA16F), specular hit distance
extern "C" void dlss_rr_emu_frame(uint32_t W, uint32_t H, const RtxptRealtimeConstants* rt, float brightnessClampK, const RtxptStablePlane* planes, const uint32_t* header,
                                  const uint16_t* stableRadiance, const uint16_t* motion, const float* specHitT, uint16_t* outColor, uint32_t* outDiffAlbedo, uint32_t* outSpecAlbedo,
                                  uint16_t* outNormalsRoughness, uint16_t* outSpecMotion)
{
    LaunchParams p = frameParams(W, H, rt, const_cast<RtxptStablePlane*>(planes), const_cast<uint32_t*>(header), reinterpret_cast<uint2*>(const_cast<uint16_t*>(stableRadiance)),
                                 reinterpret_cast<uint2*>(const_cast<uint16_t*>(motion)), const_cast<float*>(specHitT));
    p.outputColor = reinterpret_cast<uint2*>(outColor);
    const DlssRrTargets rr{ outDiffAlbedo, outSpecAlbedo, reinterpret_cast<uint2*>(outNormalsRoughness), reinterpret_cast<uint*>(outSpecMotion), brightnessClampK };
    for (uint32_t y = 0; y < H; y++) for (uint32_t x = 0; x < W; x++) dnPrepareDlssRrPixel(p, rr, (x << 16) | y);
}
