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

// ---- DENOISER_DLSS_RR (PostProcess.hlsl:198-411): the images RTXPT hands DLSS Ray Reconstruction (TagResourcesDLSSRR, Sample.cpp:2710-2757) ----------------------------------
// Formats (RenderTargets.cpp:185-197): OutputColor RGBA16F (p.outputColor), RRDiffuseAlbedo / RRSpecAlbedo R11G11B10_FLOAT, RRNormalsAndRoughness RGBA16F, RRSpecMotionVectors RG16F.
// The targets reach k_dn_prepare_dlss_rr as an argument of their own, so that LaunchParams, and with it every other kernel, keeps its layout.
struct DlssRrTargets { uint* diffAlbedo; uint* specAlbedo; uint2* normalsRoughness; uint* specMotionVectors; float brightnessClampK; };

// what the pass computes for a pixel before the stores convert it; specMotionFromGuide: the pixel keeps u_MotionVectors.xy, whose fp16 halves are stored as they are
struct DlssRrPixel { float3 color, diffAlbedo, specAlbedo, normal; float roughness; float2 specMotion; bool specMotionFromGuide; };

// ComputeSpecularMotionVector (PostProcess.hlsl:94-160, the clipToWindowScale branch): the reflection hit mirrored behind a planar reflector, camera motion only
PT_HD float2 computeSpecularMotionVector(const RealtimeParams& rt, float3 primaryHitPos, float3 primaryRayDir, float3 primaryHitNormal, float3 reflectionRay)
{
    float3 principalAxis = primaryHitNormal;
    float zObj = dot3(principalAxis, reflectionRay);
    if (zObj < 0.0f) { principalAxis = -principalAxis; zObj = -zObj; }
    zObj = fmaxf(zObj, 1e-5f);
    const float3 n = principalAxis;                                 // Duff et al., "Building an Orthonormal Basis, Revisited"
    const float s = n.z < 0.0f ? -1.0f : 1.0f;
    const float a = -1.0f / (s + n.z);
    const float b = n.x * n.y * a;
    const float3 xAxis = mk3(1.0f + s * n.x * n.x * a, s * b, -s * n.x);
    const float3 yAxis = mk3(b, s + n.y * n.y * a, -n.y);
    const float3 image = mk3(dot3(xAxis, reflectionRay), dot3(yAxis, reflectionRay), -zObj);
    const float3 w = primaryHitPos + primaryRayDir * len3(image);
    const float* Q = rt.prevWorldToClipNoOffset; const float* M = rt.worldToClipNoOffset;      // float4(w, 1) x matrix
    const float qx = ((w.x * Q[0] + w.y * Q[4]) + w.z * Q[8]) + Q[12], qy = ((w.x * Q[1] + w.y * Q[5]) + w.z * Q[9]) + Q[13], qw = ((w.x * Q[3] + w.y * Q[7]) + w.z * Q[11]) + Q[15];
    const float cx = ((w.x * M[0] + w.y * M[4]) + w.z * M[8]) + M[12], cy = ((w.x * M[1] + w.y * M[5]) + w.z * M[9]) + M[13], cw = ((w.x * M[3] + w.y * M[7]) + w.z * M[11]) + M[15];
    return mk2((qx / qw - cx / cw) * rt.clipToWindowScale[0], (qy / qw - cy / cw) * rt.clipToWindowScale[1]);
}

// DENOISER_DLSS_RR for pixel `id`, in the shader's order of operations (MIX_STABLE_RADIANCE, MIX_BY_THROUGHPUT and ALLOW_MIX_NORMALS on, as RTXPT ships it)
PT_HD DlssRrPixel dlssRrPixel(const LaunchParams& p, const uint id, const float brightnessClampK)
{
    const size_t o = pixelOffset(p, id);
    const uint planeCount = p.rt.activePlaneCount, dominant = headerWord(p, id, 3) & 3u;
    DlssRrPixel r;
    const uint2 sr = p.rt.stableRadiance[o];
    r.color = mk3(f16tof32(sr.x), f16tof32(sr.x >> 16), f16tof32(sr.y));
    float3 stableAlbedo;
    {   // sqrt(ReinhardMax(stable radiance)) (Utils.hlsli:85-90)
        const float m = fmaxf(1e-7f, fmaxf(fmaxf(r.color.x, r.color.y), r.color.z));
        const float reinhard = m / (m + 1);
        const float3 t = r.color * (reinhard / m);
        stableAlbedo = mk3(sqrtf(t.x), sqrtf(t.y), sqrtf(t.z));
    }
    const float stableAlbedoAvg = average(stableAlbedo);
    float3 guideNormals = mk3(0.0f, 0.0f, 1e-6f), diffAlbedo = mk3(0.0f), specAlbedo = mk3(0.0f);
    float roughness = 0.0f;
    float w[3];
    {   // plane weights: throughput 0.2, equalisation 0.01, dominant plane +0.05; planes without a branch drop out (plane 0 always counts), then normalised
        float thp[3] = { 1.0f, 0.0f, 0.0f }, available[3] = { 1.0f, 0.0f, 0.0f };
        for (uint i = 1; i < planeCount; i++)
        {
            if (headerWord(p, id, i) == kInvalidBranchID) continue;
            const uint4 r2 = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, i))[2];
            const float weight = sat(average(mk3(f16tof32(r2.x >> 16), f16tof32(r2.y >> 16), f16tof32(r2.z >> 16))));
            thp[i] = weight; thp[0] = sat(thp[0] - weight); available[i] = 1.0f;
        }
        for (int k = 0; k < 3; k++) w[k] = (0.0f + thp[k] * 0.2f) + 0.01f;
        if (dominant < 3u) w[dominant] += 0.05f;
        for (int k = 0; k < 3; k++) w[k] *= available[k];
        const float sum = w[0] + w[1] + w[2];
        for (int k = 0; k < 3; k++) w[k] /= sum;
    }
    for (uint i = 0; i < planeCount; i++)
    {
        if (headerWord(p, id, i) == kInvalidBranchID) continue;
        const uint4* rec = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, i));
        if (!isfinite(bitsToFloat(rec[1].w))) continue;                                     // skip sky
        const uint4 r4 = rec[4];
        r.color = r.color + mk3(f16tof32(r4.x), f16tof32(r4.x >> 16), f16tof32(r4.y));
        const float weight = w[i];
        if (weight > 1e-6f)
        {
            const uint4 r2 = rec[2], r3 = rec[3];
            guideNormals = guideNormals + weight * octUnorm32ToDir(r3.w);
            roughness = roughness + weight * f16tof32(r2.w);
            diffAlbedo = diffAlbedo + weight * mk3(f16tof32(r3.x >> 16), f16tof32(r3.y >> 16), f16tof32(r3.z >> 16));
            specAlbedo = specAlbedo + weight * mk3(f16tof32(r3.x), f16tof32(r3.y), f16tof32(r3.z));
        }
    }
    const float3 stableAlbedoGreyMix = lerp3(stableAlbedo, mk3(0.5f), 0.2f);
    diffAlbedo = lerp3(diffAlbedo, stableAlbedoGreyMix, stableAlbedoAvg / (average(diffAlbedo) + sqrtf(stableAlbedoAvg) + 1e-7f));
    const float guideNormalsLength = len3(guideNormals);
    r.normal = guideNormalsLength < 1e-5f ? mk3(0.0f, 0.0f, 1.0f) : mk3(guideNormals.x / guideNormalsLength, guideNormals.y / guideNormalsLength, guideNormals.z / guideNormalsLength);
    if (average(diffAlbedo + specAlbedo) < 0.05f) diffAlbedo = diffAlbedo + mk3(0.05f);
    const float maxRadiance = maxComp(r.color);
    if (maxRadiance > brightnessClampK) r.color = r.color * (brightnessClampK / maxRadiance);
    r.diffAlbedo = diffAlbedo; r.specAlbedo = specAlbedo; r.roughness = roughness;
    {   // specular motion vectors from plane 0's hit and the specular hit distance; the roughness test reads the mixed guide roughness
        const uint4* rec = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, 0));
        const uint4 r0 = rec[0], r1 = rec[1];
        const float3 rayOrigin = mk3(bitsToFloat(r0.x), bitsToFloat(r0.y), bitsToFloat(r0.z)), rayDir = mk3(bitsToFloat(r1.x), bitsToFloat(r1.y), bitsToFloat(r1.z));
        const float3 primaryHitPos = rayOrigin + rayDir * bitsToFloat(r1.w);
        const float3 normal = octUnorm32ToDir(rec[3].w);
        const float specHitT = p.rt.specularHitT[o];
        const float3 reflectionRay = (rayDir - (2.0f * dot3(normal, rayDir)) * normal) * specHitT;       // reflect(dir, normal) * specHitT
        r.specMotionFromGuide = !(specHitT > 1e-3f && roughness < 0.25f);                          // PathTracer::kSpecularRoughnessThreshold
        if (r.specMotionFromGuide) { const uint g = p.motionVectors[o].x; r.specMotion = mk2(f16tof32(g), f16tof32(g >> 16)); }
        else r.specMotion = computeSpecularMotionVector(p.rt, primaryHitPos, rayDir, normal, reflectionRay);
    }
    return r;
}

// the pass's stores.  R11G11B10: packR11G11B10, the rounding of every R11G11B10 store in the library; no reference source pins the conversion the hardware does on a UAV store
PT_HD void dnPrepareDlssRrPixel(const LaunchParams& p, const DlssRrTargets& rr, const uint id)
{
    const DlssRrPixel r = dlssRrPixel(p, id, rr.brightnessClampK);
    const size_t o = pixelOffset(p, id);
    p.outputColor[o] = packRGBA16F(r.color.x, r.color.y, r.color.z, 1.0f);
    rr.diffAlbedo[o] = packR11G11B10(r.diffAlbedo);
    rr.specAlbedo[o] = packR11G11B10(r.specAlbedo);
    rr.normalsRoughness[o] = packRGBA16F(r.normal.x, r.normal.y, r.normal.z, r.roughness);
    rr.specMotionVectors[o] = r.specMotionFromGuide ? p.motionVectors[o].x : (f32tof16(r.specMotion.x) | (f32tof16(r.specMotion.y) << 16));
}

} // namespace pt
