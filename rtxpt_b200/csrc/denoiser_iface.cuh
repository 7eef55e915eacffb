// denoiser_iface.cuh - RTXPT's side of the denoiser interface (SURVEY §8 row a18) as __host__ __device__ pixel bodies: PostProcess.hlsl DENOISER_PREPARE_INPUTS (ReBLUR variant,
// ProcessingPasses/PostProcess.hlsl:444-570) and DENOISER_FINAL_MERGE (:577-690) with NRD's front / back-end packing (External/Nrd/Shaders/Include/NRD.hlsli:333-381, :526-529,
// :646-677, :728-750, :869-874).  Kernels: realtime_kernels.cu; host build for the CPU parity test: tests/emu.
#pragma once
#include "wavefront.cuh"
#include "debug_views.cuh"

namespace pt {

PT_HD uint2 packRGBA16F(float x, float y, float z, float w) { return make_uint2(f32tof16(x) | (f32tof16(y) << 16), f32tof16(z) | (f32tof16(w) << 16)); }
PT_HD unsigned char unorm8(float v) { return (unsigned char)(sat(v) * 255.0f + 0.5f); }
PT_HD float3 linearToYCoCg(float3 c) { return mk3(dot3(c, mk3(0.25f, 0.5f, 0.25f)), dot3(c, mk3(0.5f, 0.0f, -0.5f)), dot3(c, mk3(-0.25f, 0.5f, -0.25f))); }
PT_HD float3 yCoCgToLinear(float3 c) { const float t = c.x - c.z; return mk3(fmaxf(t + c.y, 0.f), fmaxf(c.x + c.z, 0.f), fmaxf(t - c.y, 0.f)); }
PT_HD void nrdRadianceClamp(float3& radiance, float preExposedGrayLuminance, float rangeK)
{
    const float clampMax = fminf(255.0f, preExposedGrayLuminance * rangeK);
    const float lum = luminance(radiance);
    if (lum > clampMax) radiance = radiance * (clampMax / lum);
}
PT_HD uint2 packRadianceAndNormHitDist(float3 radiance, float normHitDist)      // REBLUR_FrontEnd_PackRadianceAndNormHitDist(sanitize = true)
{
    const bool invalid = !isfinite(radiance.x) || !isfinite(radiance.y) || !isfinite(radiance.z);
    radiance = invalid ? mk3(0.f) : mk3(clampf(radiance.x, 0.f, 65504.0f), clampf(radiance.y, 0.f, 65504.0f), clampf(radiance.z, 0.f, 65504.0f));
    normHitDist = isfinite(normHitDist) ? sat(normHitDist) : 0.0f;
    const float3 y = linearToYCoCg(radiance);
    return packRGBA16F(y.x, y.y, y.z, normHitDist);
}


// DENOISER_PREPARE_INPUTS for pixel `id` ((x << 16) | y) of stable plane p.rt.dnPlane
PT_HD void dnPrepareInputsPixel(const LaunchParams& p, const uint id)
{

    const uint plane = p.rt.dnPlane;
        {

        const size_t o = pixelOffset(p, id);
        if (p.rt.dnInitWithStableRadiance)
        {
            const uint2 sr = p.rt.stableRadiance[o];
            p.outputColor[o] = make_uint2(sr.x, (sr.y & 0xFFFFu) | (0x3C00u << 16));        // float4(stable radiance, 1)
            p.rt.dnHistoryClampRelax[o] = 0;
        }
        bool hasSurface = false;
        const uint branchID = headerWord(p, id, plane);
        if (branchID != kInvalidBranchID)
        {
            const uint4* rec = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, plane));
            const uint4 r1 = rec[1], r2 = rec[2], r3 = rec[3], r4 = rec[4];
            const float sceneLength = bitsToFloat(r1.w);
            if (isfinite(sceneLength))
            {
                hasSurface = true;
                const float3 diffEstimate = mk3(f16tof32(r3.x >> 16), f16tof32(r3.y >> 16), f16tof32(r3.z >> 16)), specEstimate = mk3(f16tof32(r3.x), f16tof32(r3.y), f16tof32(r3.z));
                float3 co, cd; computeCameraRay(p.c, id, p.c.sampleBaseIndex, co, cd);
                const float3 vp = co + cd * sceneLength;
                const float* M = p.rt.dn.matWorldToView;
                const float viewZ = ((vp.x * M[2] + vp.y * M[6]) + vp.z * M[10]) + M[14];
                const float3 thp = mk3(f16tof32(r2.x >> 16), f16tof32(r2.y >> 16), f16tof32(r2.z >> 16));
                p.rt.dnViewZ[o] = viewZ;
                p.rt.dnMotion[o] = make_uint2((r2.x & 0xFFFFu) | (r2.y << 16), r2.z & 0xFFFFu);       // float4(motionVectors, 0): the fp16 halves move as they are
                const float spRoughness = f16tof32(r2.w);
                float finalRoughness = fmaxf(0.2f, spRoughness);
                float specularSuppressionMul = 1.0f;
                if (plane == 0 && p.rt.dn.stablePlanesSuppressPrimaryIndirectSpecularK != 0.0f && p.rt.activePlaneCount > 1)
                {
                    bool shouldSuppress = true;
                    for (uint i = 1; i < p.rt.activePlaneCount; i++) shouldSuppress = shouldSuppress && headerWord(p, id, i) != kInvalidBranchID;
                    if (shouldSuppress) specularSuppressionMul = sat(1 - p.rt.dn.stablePlanesSuppressPrimaryIndirectSpecularK);
                }
                const float3 normal = octUnorm32ToDir(r3.w);
                float disocclusionRelax = 0.0f;
                if (vertexIndexFromBranchID(branchID) > 1)
                {   // ComputeDisocclusionRelaxation: how far the plane's (virtual) normal turns towards the four neighbours
                    const int px = int(id >> 16), py = int(id & 0xFFFFu);
                    const int ox[4] = { -1, 1, 0, 0 }, oy[4] = { 0, 0, -1, 1 };
                    #pragma unroll
                    for (int n = 0; n < 4; n++)
                    {
                        const uint nx = uint(min(max(px + ox[n], 0), int(p.c.imageWidth) - 1)), ny = uint(min(max(py + oy[n], 0), int(p.c.imageHeight) - 1));
                        const uint nid = (nx << 16) | ny;
                        if (headerWord(p, nid, plane) == kInvalidBranchID) disocclusionRelax += 0.02f;
                        else disocclusionRelax += 1 - dot3(normal, octUnorm32ToDir(p.rt.planes[planeAddress(p.rt, nid, plane)].PackedNormal));
                    }
                    disocclusionRelax = sat((disocclusionRelax - 0.00002f) * 25);
                }
                p.rt.dnDisocclusionMix[o] = unorm8(disocclusionRelax);
                p.rt.dnHistoryClampRelax[o] = unorm8(sat(float(p.rt.dnHistoryClampRelax[o]) / 255.0f + disocclusionRelax * sat(luminance(thp))));
                finalRoughness = sat(finalRoughness + disocclusionRelax);
                // StablePlane::GetNoisyDiffRadiance / GetNoisySpecRadiance
                const float3 l = mk3(f16tof32(r4.x), f16tof32(r4.x >> 16), f16tof32(r4.y)); const float specAvg = f16tof32(r4.y >> 16), totalAvg = average(l);
                float3 diff = l * sat(1.0f - specAvg / (totalAvg + 1e-12f)), spec = l * sat(specAvg / (totalAvg + 1e-12f));
                diff = diff / diffEstimate; spec = spec / specEstimate;
                spec = spec * specularSuppressionMul;
                {   // NRD_FrontEnd_PackNormalAndRoughness, R10G10B10A2_UNORM, linear roughness, material ID 0
                    float3 v = normal / (fabsf(normal.x) + fabsf(normal.y) + fabsf(normal.z));
                    const float wx = (1.0f - fabsf(v.y)) * (v.x >= 0.0f ? 1.0f : -1.0f), wy = (1.0f - fabsf(v.x)) * (v.y >= 0.0f ? 1.0f : -1.0f);
                    const float ex = (v.z >= 0.0f ? v.x : wx) * 0.5f + 0.5f, ey = (v.z >= 0.0f ? v.y : wy) * 0.5f + 0.5f;
                    p.rt.dnNormalRoughness[o] = uint(sat(ex) * 1023.0f + 0.5f) | (uint(sat(ey) * 1023.0f + 0.5f) << 10) | (uint(sat(finalRoughness) * 1023.0f + 0.5f) << 20);
                }
                nrdRadianceClamp(diff, p.rt.dn.preExposedGrayLuminance, p.rt.dn.denoiserRadianceClampK * 16); nrdRadianceClamp(spec, p.rt.dn.preExposedGrayLuminance, p.rt.dn.denoiserRadianceClampK * 16);
                float specHitT = 0;
                if ((headerWord(p, id, 3) & 3u) == plane) specHitT = p.rt.specularHitT[o];
                p.rt.dnDiff[o] = packRadianceAndNormHitDist(diff, 0.0f);
                const float* hp = p.rt.dn.hitDistanceParameters;
                const float f = (hp[0] + fabsf(viewZ) * hp[1]) * lerpf(1.0f, hp[2], sat(exp2f(hp[3] * spRoughness * spRoughness)));     // _REBLUR_GetHitDistanceNormalization
                p.rt.dnSpec[o] = packRadianceAndNormHitDist(spec, sat(specHitT / f));
            }
        }
        if (!hasSurface) p.rt.dnViewZ[o] = 3.402823466e+38f;         // VIEWZ_SKY_MARKER
        }
}

// DENOISER_FINAL_MERGE for pixel `id`
PT_HD void dnFinalMergePixel(const LaunchParams& p, const uint id)
{

        const size_t o = pixelOffset(p, id);
        if (p.rt.dnViewZ[o] == 3.402823466e+38f) return;
        const uint4 r3 = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, p.rt.dnPlane))[3];
        const float3 diffEstimate = mk3(f16tof32(r3.x >> 16), f16tof32(r3.y >> 16), f16tof32(r3.z >> 16)), specEstimate = mk3(f16tof32(r3.x), f16tof32(r3.y), f16tof32(r3.z));
        const uint2 dd = p.rt.dnDenoisedDiff[o], ds = p.rt.dnDenoisedSpec[o];
        const float3 diff = yCoCgToLinear(mk3(f16tof32(dd.x), f16tof32(dd.x >> 16), f16tof32(dd.y))) * diffEstimate;
        const float3 spec = yCoCgToLinear(mk3(f16tof32(ds.x), f16tof32(ds.x >> 16), f16tof32(ds.y))) * specEstimate;
        const float3 sum = mk3(fmaxf(diff.x + spec.x, 0.f), fmaxf(diff.y + spec.y, 0.f), fmaxf(diff.z + spec.z, 0.f));
        const uint2 c = p.outputColor[o];
        p.outputColor[o] = make_uint2(f32tof16(f16tof32(c.x) + sum.x) | (f32tof16(f16tof32(c.x >> 16) + sum.y) << 16), f32tof16(f16tof32(c.y) + sum.z) | (c.y & 0xFFFF0000u));
    }

// the denoiser-merge debug views of the merged plane (PostProcess.hlsl:633-681, rtxpt_b200_set_debug_view): the same inputs as dnFinalMergePixel, read again
PT_HD void dnFinalMergeDebugPixel(const LaunchParams& p, const uint id)
{
    const uint px = id >> 16, py = id & 0xFFFFu, W = p.c.imageWidth, H = p.c.imageHeight;
    const size_t o = pixelOffset(p, id);
    const uint4* rec = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, p.rt.dnPlane));
    if (mergeDebugChecker(p.dbg.planeIndex, p.rt.dnPlane, px, py, W, H, p.rt.activePlaneCount)) { const float c = float((px + py) % 2u); p.dbg.viz[o] = packDebugPixel(make_float4(c, c, c, 1.0f)); }
    uint tx, ty;
    if (!mergeDebugTarget(p.dbg.view, p.dbg.planeIndex, p.rt.dnPlane, px, py, W, H, tx, ty)) return;
    MergeDebugInputs m;
    m.viewZ = p.rt.dnViewZ[o];
    m.relaxedDisocclusion = 0.0f; m.diff = mk3(0.0f); m.spec = mk3(0.0f);
    if (m.viewZ != 3.402823466e+38f)
    {
        const uint4 r3 = rec[3];
        const float3 diffEstimate = mk3(f16tof32(r3.x >> 16), f16tof32(r3.y >> 16), f16tof32(r3.z >> 16)), specEstimate = mk3(f16tof32(r3.x), f16tof32(r3.y), f16tof32(r3.z));
        const uint2 dd = p.rt.dnDenoisedDiff[o], ds = p.rt.dnDenoisedSpec[o];
        m.diff = yCoCgToLinear(mk3(f16tof32(dd.x), f16tof32(dd.x >> 16), f16tof32(dd.y))) * diffEstimate;
        m.spec = yCoCgToLinear(mk3(f16tof32(ds.x), f16tof32(ds.x >> 16), f16tof32(ds.y))) * specEstimate;
        m.relaxedDisocclusion = float(p.rt.dnDisocclusionMix[o]) / 255.0f;             // R8_UNORM
    }
    const uint4 r2 = rec[2];                                                              // PackedThpAndMVs: throughput in the high halves
    m.throughput = mk3(f16tof32(r2.x >> 16), f16tof32(r2.y >> 16), f16tof32(r2.z >> 16));
    p.dbg.viz[size_t(ty) * W + tx] = packDebugPixel(mergeDebugColor(p.dbg.view, m));
}

} // namespace pt
