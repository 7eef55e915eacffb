// reblur_passes.cuh - the per-pixel bodies of the ReBLUR passes as __host__ __device__ functions: reblur_kernels.cu wraps each in a kernel (one thread per pixel); the
// test-only host build tests/emu/reblur_host_emu.cu runs the very same source pixel by pixel on the CPU so that the port can be checked against the oracle without a GPU.
// NRD's REBLUR_DIFFUSE_SPECULAR chain for one stable plane (SURVEY §8 row a18 / K9), pass by pass along the dispatch graph
// (External/Nrd/Source/Denoisers/Reblur_DiffuseSpecular.hpp:71-270) in RTXPT's configuration (Rtxpt/NRD/NrdConfig.cpp:49-61, NrdIntegration.cpp:375-408):
//   beyondDenoisingRange            REBLUR_ClassifyTiles.cs.hlsl:21-60 (the per-texel predicate; the kernel counts it over a 16x16 tile)
//   hitDistReconstructionPixel      REBLUR_HitDistReconstruction.hlsli:11-155 (5x5 or 3x3)
//   spatialPixel<PRE|BLUR|POST>     REBLUR_PrePass / REBLUR_Blur / REBLUR_PostBlur.hlsli + REBLUR_Common_{Diffuse,Specular}SpatialFilter.hlsli
//   temporalAccumulationPixel       REBLUR_TemporalAccumulation.hlsli:11-937
//   historyFixPixel                 REBLUR_HistoryFix.hlsli:11-496
//   temporalStabilizationPixel      REBLUR_TemporalStabilization.hlsli:11-369
// Every pass reads only buffers no thread of the same pass writes (except its own pixel), so thread order does not matter.
#pragma once
#include "reblur.cuh"

namespace pt { namespace rb {


// SKY: statement run for pixels the pass skips (sky tiles and pixels beyond the denoising range); `pix` is in scope
#define RB_PIXEL_PROLOGUE_SKY(SKY) \
    const size_t pix = size_t(y) * p.W + x; \
    const float viewZ = fabsf(p.viewZ[pix] * p.viewZScale); \
    if (p.tiles[size_t(y >> 4) * p.tilesW + (x >> 4)] || viewZ > p.denoisingRange) { SKY; return; } \
    const int W = int(p.W), H = int(p.H); \
    const float2 rectSizeInv = mk2(1.0f / float(W), 1.0f / float(H)); \
    const float2 pixelUv = mk2((float(x) + 0.5f) * rectSizeInv.x, (float(y) + 0.5f) * rectSizeInv.y)
#define RB_PIXEL_PROLOGUE RB_PIXEL_PROLOGUE_SKY((void)0)

PT_HD float viewZAt(const Params& p, int x, int y) { return fabsf(p.viewZ[size_t(y) * p.W + x] * p.viewZScale); }
PT_HD bool inScreen(float2 uv) { return uv.x > 0.0f && uv.y > 0.0f && uv.x < 1.0f && uv.y < 1.0f; }
// g_Special8: 8 taps on two rings, .z = the radius fed to the Gaussian (REBLUR_Common.hlsli Poisson table replacement); the loops over it are fully unrolled, so it folds to immediates
PT_HD float3 special8(int n)
{
    const float t[8][3] = { { -1, 0, 1 }, { 0, 1, 1 }, { 1, 0, 1 }, { 0, -1, 1 }, { -0.35355339f, 0.35355339f, 0.5f }, { 0.35355339f, 0.35355339f, 0.5f }, { 0.35355339f, -0.35355339f, 0.5f }, { -0.35355339f, -0.35355339f, 0.5f } };
    return mk3(t[n][0], t[n][1], t[n][2]);
}

// ---- ClassifyTiles ---------------------------------------------------------------------------------------------------------------------------------------------
PT_HD bool beyondDenoisingRange(const Params& p, int x, int y)
{   // out-of-bounds texels read 0: partial border tiles are never sky
    const float z = (x < int(p.W) && y < int(p.H)) ? viewZAt(p, x, y) : 0.0f;
    return z > p.denoisingRange;
}

// ---- HitDistReconstruction 5x5 / 3x3: in -> tmp2 (which images those are: routeFrame, reblur_host.h) ------------------------------------------------------------------------------------------------------------------------
// The 5x5 neighbourhood comes through a tap source: straight from global memory (GlobalTaps: the host build and the border tiles' fallback) or from the CTA's shared-memory
// tile (reblur_kernels.cu: viewZ, the UNPACKED normal / roughness and the two hit distances of the 20x20 region staged by TMA) - what NRD's PRELOAD_INTO_SMEM does for the same
// pass (External/Nrd/Shaders/Include/Common.hlsli:143-175): the saving is the 24 normal unpacks and clamped address computations per pixel, not bandwidth.
struct GlobalTaps
{
    const Params& p; int W, H;
    PT_HD float viewZ(int qx, int qy) const { return viewZAt(p, qx, qy); }                     // callers pass clamped coordinates
    PT_HD float4 normalRoughness(int qx, int qy) const { float m; return unpackNormalRoughness(p.normalRoughness[size_t(qy) * W + qx], m); }
    PT_HD float diffHitDist(int qx, int qy) const { return f16tof32(p.inDiff[size_t(qy) * W + qx].y >> 16); }
    PT_HD float specHitDist(int qx, int qy) const { return f16tof32(p.inSpec[size_t(qy) * W + qx].y >> 16); }
};
// RADIUS 2: REBLUR_DiffuseSpecular_HitDistReconstruction_5x5.cs.hlsl (NRD_USE_BORDER_2); RADIUS 1: REBLUR_DiffuseSpecular_HitDistReconstruction.cs.hlsl (AREA_3X3, BORDER 1) - the same body
template <int RADIUS, typename Taps>
PT_HD void hitDistReconstructionBody(const Params& p, const int x, const int y, const Taps& taps)
{
    RB_PIXEL_PROLOGUE;
    float mid; const float4 nr = unpackNormalRoughness(p.normalRoughness[pix], mid);
    const float3 N = xyz(nr), Nv = worldToViewRotate(p, N); const float roughness = nr.w;
    const float3 Xv = reconstructViewPosition(p.frustum, pixelUv, viewZ);
    const float2 gw = geometryWeightParams(p, frustumSize(p, viewZ), Xv, Nv), rw = relaxedRoughnessWeightParams(roughness * roughness, 1.0f, 0.01f);
    const float diffNormalW = normalWeightParam(1.0f, 1.0f, 1.0f), specNormalW = normalWeightParam(1.0f, 1.0f, roughness);
    const float4 d = unpackRGBA16F(p.inDiff[pix]), s = unpackRGBA16F(p.inSpec[pix]);
    float cx = d.w, cy = s.w, sx = cx != 0.0f ? 1000.0f : 0.0f, sy = cy != 0.0f ? 1000.0f : 0.0f;
    cx *= sx; cy *= sy;
    for (int j = -RADIUS; j <= RADIUS; j++) for (int i = -RADIUS; i <= RADIUS; i++)
    {
        if (i == 0 && j == 0) continue;
        const int qx = clampi(x + i, 0, W - 1), qy = clampi(y + j, 0, H - 1);
        const float2 uv = mk2(pixelUv.x + float(i) * rectSizeInv.x, pixelUv.y + float(j) * rectSizeInv.y);
        float w = inScreen(uv) ? 1.0f : 0.0f;
        w *= gaussianWeight(sqrtf(float(i * i + j * j)) * 0.5f);
        w *= weight(dot3(Nv, reconstructViewPosition(p.frustum, uv, taps.viewZ(qx, qy))), gw.x, gw.y);
        const float4 ns = taps.normalRoughness(qx, qy);
        const float angle = acosApprox(dot3(N, xyz(ns)));
        float wx = w * exponentialWeight(angle, diffNormalW, 0.0f), wy = w * exponentialWeight(angle, specNormalW, 0.0f) * exponentialWeight(ns.w * ns.w, rw.x, rw.y);
        float dx = taps.diffHitDist(qx, qy), dy = taps.specHitDist(qx, qy);
        if (wx == 0.0f) dx = 0.0f; if (wy == 0.0f) dy = 0.0f;
        wx = dx != 0.0f ? wx : 0.0f; wy = dy != 0.0f ? wy : 0.0f;
        cx += dx * wx; cy += dy * wy; sx += wx; sy += wy;
    }
    cx /= fmaxf(sx, kEps); cy /= fmaxf(sy, kEps);
    p.tmp2Diff[pix] = packRGBA16F(make_float4(d.x, d.y, d.z, cx)); p.tmp2Spec[pix] = packRGBA16F(make_float4(s.x, s.y, s.z, cy));
}
template <int RADIUS = 2>
PT_HD void hitDistReconstructionPixel(const Params& p, const int x, const int y) { const GlobalTaps t{ p, int(p.W), int(p.H) }; hitDistReconstructionBody<RADIUS>(p, x, y, t); }

// ---- spatial passes ----------------------------------------------------------------------------------------------------------------------------------------------------
// MODE 0 PrePass: tmp2 -> tmp1 (+ hit distance for tracking); 1 Blur: tmp1 -> tmp2 (+ viewZ copy into the history); 2 PostBlur: tmp2 -> history (+ normal/roughness copy)
template <int MODE>
PT_HD void spatialPixel(const Params& p, const int x, const int y)
{
    if (MODE == 1)
    {   // Blur copies viewZ for the next frame, sky included, before any early out
        p.prevViewZ[size_t(y) * p.W + x] = p.viewZ[size_t(y) * p.W + x];
    }
    if (MODE == 2)
    {   // PostBlur copies the packed normal / roughness for the next frame
        p.prevNormalRoughness[size_t(y) * p.W + x] = p.normalRoughness[size_t(y) * p.W + x];
    }
    RB_PIXEL_PROLOGUE_SKY(if (MODE == 0) p.trackingTransient[pix] = 0);
    const uint2* srcDiff = MODE == 1 ? p.tmp1Diff : p.tmp2Diff; const uint2* srcSpec = MODE == 1 ? p.tmp1Spec : p.tmp2Spec;
    uint2* dstDiff = MODE == 0 ? p.tmp1Diff : (MODE == 1 ? p.tmp2Diff : p.diffHistory); uint2* dstSpec = MODE == 0 ? p.tmp1Spec : (MODE == 1 ? p.tmp2Spec : p.specHistory);
    const float fractionScale = MODE == 0 ? 2.0f : (MODE == 1 ? 1.0f : 0.5f), radiusScale = MODE == 2 ? 2.0f : 1.0f;
    const Rotator baseRotator = MODE == 0 ? p.rotatorPre : (MODE == 1 ? p.rotator : p.rotatorPost);
    float materialID; const float4 nr = unpackNormalRoughness(p.normalRoughness[pix], materialID);
    const float3 N = xyz(nr), Nv = worldToViewRotate(p, N); const float roughness = nr.w;
    const float3 Xv = reconstructViewPosition(p.frustum, pixelUv, viewZ), Vv = norm3(-Xv);
    const float NoV = fabsf(dot3(Nv, Vv)), fs = frustumSize(p, viewZ);
    float2 d1 = mk2(0.f, 0.f);
    if (MODE != 0) { const uchar2 q = p.data1[pix]; d1 = mk2(float(q.x) / 255.0f * 63.0f, float(q.y) / 255.0f * 63.0f); }
    // ---- diffuse: screen-space Poisson kernel ----
    {
        float sum = 1.0f; float4 diff = unpackRGBA16F(srcDiff[pix]);
        if (MODE != 0 || p.diffPrepassBlurRadius != 0.0f)
        {
            const float hitDist = diff.w * hitDistanceNormalization(p, viewZ, 1.0f), hitDistFactor = sat(hitDist / fs);
            float nl, blurRadius, areaFactor;
            if (MODE == 0) { nl = 1.0f / 11.0f; blurRadius = p.diffPrepassBlurRadius; areaFactor = hitDistFactor; }
            else { const float boost = (1.0f - fadeBasedOnAccumulatedFrames(p, d1.x)) * (1.0f - pow5(NoV)); nl = 1.0f / (1.0f + (1.0f - boost) * d1.x); blurRadius = p.maxBlurRadius; areaFactor = hitDistFactor * nl; }
            blurRadius = fmaxf(blurRadius * sqrt01(areaFactor) * radiusScale, p.minBlurRadius);
            const float2 gw = geometryWeightParams(p, fs, Xv, Nv), hw = hitDistanceWeightParams(diff.w, nl, 1.0f);
            const float normalW = normalWeightParam(nl, p.lobeAngleFraction, 1.0f) / fractionScale;
            float minHitDistWeight = p.minHitDistanceWeight * fractionScale; if (MODE != 0) minHitDistWeight *= sqrtf(nl);
            float2 skew = mk2(1.f, 1.f);
            if (MODE != 0) { skew = mk2(lerpf(1.0f - fabsf(Nv.x), 1.0f, NoV), lerpf(1.0f - fabsf(Nv.y), 1.0f, NoV)); const float m = fmaxf(skew.x, skew.y); skew = mk2(skew.x / m, skew.y / m); }
            const Rotator scaled = scaleRotator(baseRotator, mk2(skew.x * rectSizeInv.x * blurRadius, skew.y * rectSizeInv.y * blurRadius));
            #pragma unroll
            for (int n = 0; n < 8; n++)
            {
                const float2 o = rotate(scaled, mk2(special8(n).x, special8(n).y));
                const float2 uv = mk2((floorf((pixelUv.x + o.x) * float(W)) + 0.5f) * rectSizeInv.x, (floorf((pixelUv.y + o.y) * float(H)) + 0.5f) * rectSizeInv.y);
                const int qx = clampi(int(floorf(fminf(uv.x, 1.0f - 0.5f * rectSizeInv.x) * float(W))), 0, W - 1), qy = clampi(int(floorf(fminf(uv.y, 1.0f - 0.5f * rectSizeInv.y) * float(H))), 0, H - 1);
                const size_t q = size_t(qy) * W + qx;
                float ms; const float4 Ns = unpackNormalRoughness(p.normalRoughness[q], ms);
                float w = inScreen(uv) ? 1.0f : 0.0f;
                w *= weight(dot3(Nv, reconstructViewPosition(p.frustum, uv, viewZAt(p, qx, qy))), gw.x, gw.y);
                w *= compareMaterials(materialID, ms, p.minMaterialDiff) ? 1.0f : 0.0f;
                w *= weight(acosApprox(dot3(N, xyz(Ns))), normalW, 0.0f);
                float4 sv = unpackRGBA16F(srcDiff[q]); if (w == 0.0f) sv = make_float4(0, 0, 0, 0);
                w *= lerpf(minHitDistWeight, 1.0f, exponentialWeight(sv.w, hw.x, hw.y));
                w *= gaussianWeight(special8(n).z);
                sum += w; diff = diff + sv * w;
            }
            diff = diff * positiveRcp(sum);
        }
        dstDiff[pix] = packRGBA16F(diff);
    }
    // ---- specular: screen space in the pre-pass, world-space kernel bent towards the dominant direction afterwards ----
    {
        float sum = 1.0f; float4 spec = unpackRGBA16F(srcSpec[pix]);
        const float smc = specMagicCurve(roughness);
        if (MODE != 0 || p.specPrepassBlurRadius != 0.0f)
        {
            Rng rng; rng.init(uint(x), uint(y), p.frameIndex);
            const float4 Dv = specularDominantDirection(Nv, Vv, roughness);
            const float NoD = fabsf(dot3(Nv, xyz(Dv)));
            const float hitDist = spec.w * hitDistanceNormalization(p, viewZ, roughness), hitDistFactor = sat(hitDist / fs);
            float hitDistForTracking = hitDist == 0.0f ? kInf : hitDist;
            float nl, blurRadius, areaFactor;
            if (MODE == 0) { nl = 1.0f / 11.0f; blurRadius = p.specPrepassBlurRadius; areaFactor = roughness * hitDistFactor; }
            else { const float boost = (1.0f - fadeBasedOnAccumulatedFrames(p, d1.y)) * (1.0f - pow5(NoV)) * smc; nl = 1.0f / (1.0f + (1.0f - boost) * d1.y); blurRadius = p.maxBlurRadius; areaFactor = roughness * hitDistFactor * nl; }
            blurRadius *= sqrt01(areaFactor);
            if (MODE == 0) blurRadius = fminf(blurRadius, hitDist * NoD * specularLobeTanHalfAngle(roughness, 0.3f) / pixelRadiusToWorld(p, 1.0f, viewZ + hitDist * Dv.w));
            blurRadius = fmaxf(blurRadius * radiusScale, p.minBlurRadius * smc);
            const float2 gw = geometryWeightParams(p, fs, Xv, Nv), rw = roughnessWeightParams(roughness, sat(p.roughnessFraction * fractionScale)), hw = hitDistanceWeightParams(spec.w, nl, roughness);
            const float normalW = normalWeightParam(nl, p.lobeAngleFraction, roughness) / fractionScale;
            float minHitDistWeight = p.minHitDistanceWeight * fractionScale * smc; if (MODE != 0) minHitDistWeight *= sqrtf(nl);
            Rotator scaled = baseRotator; float3 Tv = mk3(0.f), Bv = mk3(0.f);
            if (MODE == 0) scaled = scaleRotator(baseRotator, mk2(rectSizeInv.x * blurRadius, rectSizeInv.y * blurRadius));
            else
            {
                const float bent = sqrtf(hitDistFactor);
                float skewFactor = lerpf(0.25f + 0.75f * roughness, 1.0f, NoD); skewFactor = lerpf(skewFactor, 1.0f, nl); skewFactor = lerpf(1.0f, skewFactor, bent);
                const float3 D = norm3(lerp3(Nv, xyz(Dv), bent));
                getBasis(Nv, Tv, Bv);
                if (fabsf(dot3(D, Nv)) < 0.999f) { const float3 R = Nv * (2.0f * dot3(Nv, D)) - D; Tv = norm3(cross3(Nv, R)); Bv = cross3(R, Tv); }
                const float worldRadius = pixelRadiusToWorld(p, blurRadius, viewZ);
                Tv = Tv * (worldRadius * skewFactor); Bv = Bv * (worldRadius / skewFactor);
            }
            #pragma unroll
            for (int n = 0; n < 8; n++)
            {
                float2 uvRaw;
                if (MODE == 0) { const float2 o = rotate(scaled, mk2(special8(n).x, special8(n).y)); uvRaw = mk2(pixelUv.x + o.x, pixelUv.y + o.y); }
                else
                {
                    const float2 o = rotate(baseRotator, mk2(special8(n).x, special8(n).y));
                    const float3 q3 = Xv + Tv * o.x + Bv * o.y; const float* M = p.viewToClip;
                    const float cx = q3.x * M[0] + q3.y * M[4] + q3.z * M[8] + M[12], cy = q3.x * M[1] + q3.y * M[5] + q3.z * M[9] + M[13], cw = q3.x * M[3] + q3.y * M[7] + q3.z * M[11] + M[15];
                    uvRaw = mk2(cx / cw * 0.5f + 0.5f, -(cy / cw) * 0.5f + 0.5f);
                }
                const float2 uv = mk2((floorf(uvRaw.x * float(W)) + 0.5f) * rectSizeInv.x, (floorf(uvRaw.y * float(H)) + 0.5f) * rectSizeInv.y);
                const int qx = clampi(int(floorf(fminf(uv.x, 1.0f - 0.5f * rectSizeInv.x) * float(W))), 0, W - 1), qy = clampi(int(floorf(fminf(uv.y, 1.0f - 0.5f * rectSizeInv.y) * float(H))), 0, H - 1);
                const size_t q = size_t(qy) * W + qx;
                const float zs = viewZAt(p, qx, qy);
                float ms; const float4 Ns = unpackNormalRoughness(p.normalRoughness[q], ms);
                const float3 Xvs = reconstructViewPosition(p.frustum, uv, zs);
                float w = inScreen(uv) ? 1.0f : 0.0f;
                w *= weight(dot3(Nv, Xvs), gw.x, gw.y);
                w *= compareMaterials(materialID, ms, p.minMaterialSpec) ? 1.0f : 0.0f;
                w *= weight(acosApprox(dot3(N, xyz(Ns))), normalW, 0.0f);
                w *= weight(Ns.w, rw.x, rw.y);
                float4 sv = unpackRGBA16F(srcSpec[q]); if (w == 0.0f) sv = make_float4(0, 0, 0, 0);
                if (MODE == 0)
                {
                    const float hs = sv.w * hitDistanceNormalization(p, zs, Ns.w);
                    if (rng.next() < w * NoV * (hs != 0.0f ? 1.0f : 0.0f)) hitDistForTracking = fminf(hitDistForTracking, hs);
                    w *= p.usePrepassOnlyForSpecularMotionEstimation ? 0.0f : 1.0f;
                    const float dd = len3(Xvs - Xv) + kEps;
                    w *= lerpf(sat(hs / (dd + hitDist)), 1.0f, linearStep(0.5f, 1.0f, roughness));
                }
                w *= lerpf(minHitDistWeight, 1.0f, exponentialWeight(sv.w, hw.x, hw.y));
                w *= gaussianWeight(special8(n).z);
                sum += w; spec = spec + sv * w;
            }
            spec = spec * positiveRcp(sum);
            if (MODE == 0) stHalf(p.trackingTransient, pix, hitDistForTracking == kInf ? 0.0f : hitDistForTracking);
        }
        dstSpec[pix] = packRGBA16F(spec);
    }
}

// ---- TemporalAccumulation: tmp1 + history -> tmp2, transient fast history, tracking (current), data1, data2 -----------------------------------------------------------------
PT_HD void temporalAccumulationPixel(const Params& p, const int x, const int y)
{
    RB_PIXEL_PROLOGUE_SKY(p.trackingCurr[pix] = 0; p.diffFastTransient[pix] = 0; p.specFastTransient[pix] = 0; p.data1[pix] = make_uchar2(0, 0); p.data2[pix] = 0);      // what a freshly cleared transient pool holds
    const float2 rectSize = mk2(float(W), float(H));
    const float3 Xv = reconstructViewPosition(p.frustum, pixelUv, viewZ), X = viewToWorldRotate(p, Xv);
    const float3 cameraDelta = mk3(p.cameraDelta[0], p.cameraDelta[1], p.cameraDelta[2]);
    auto normalAt = [&](int qx, int qy) { float m; return unpackNormalRoughness(p.normalRoughness[size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)], m); };
    auto prevNormalAt = [&](int qx, int qy) { float m; return unpackNormalRoughness(p.prevNormalRoughness[size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)], m); };
    auto prevZ = [&](int qx, int qy) { return fabsf(p.prevViewZ[size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)] * p.viewZScale); };
    auto prevInternal = [&](int qx, int qy) { return uint(p.prevInternalData[size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)]); };
    auto rotatePrevInverse = [&](float3 v) { const float* t = p.worldToViewPrev; return mk3(t[0] * v.x + t[4] * v.y + t[8] * v.z, t[1] * v.x + t[5] * v.y + t[9] * v.z, t[2] * v.x + t[6] * v.y + t[10] * v.z); };
    auto inScreenBilinear = [&](float2 o) { const float ax = (o.x >= 0.0f && o.x < rectSize.x) ? 1.0f : 0.0f, ay = (o.y >= 0.0f && o.y < rectSize.y) ? 1.0f : 0.0f, bx = (o.x + 1 >= 0.0f && o.x + 1 < rectSize.x) ? 1.0f : 0.0f, by = (o.y + 1 >= 0.0f && o.y + 1 < rectSize.y) ? 1.0f : 0.0f;
                                            return make_float4(ax * ay, bx * ay, ax * by, bx * by); };
    // 3x3: tracking distance, averaged normal of the first 2x2, roughness variance
    float3 Navg = mk3(0.f); float hitDistForTracking = kInf, rM1 = 0.f, rM2 = 0.f;
    for (int j = 0; j <= 2; j++) for (int i = 0; i <= 2; i++)
    {
        const int qx = clampi(x + i - 1, 0, W - 1), qy = clampi(y + j - 1, 0, H - 1); const size_t q = size_t(qy) * W + qx;
        const float4 n = normalAt(qx, qy);
        if (i < 2 && j < 2) Navg = Navg + xyz(n);
        const float hd = p.specPrepassBlurRadius == 0.0f ? f16tof32(p.tmp1Spec[q].y >> 16) : ldHalf(p.trackingTransient, q);
        hitDistForTracking = fminf(hitDistForTracking, hd == 0.0f ? kInf : hd);
        const float r2 = n.w * n.w; rM1 += r2; rM2 += r2 * r2;
    }
    Navg = Navg / 4.0f;
    float materialID; const float4 nrC = unpackNormalRoughness(p.normalRoughness[pix], materialID);
    const float3 N = xyz(nrC); const float roughness = nrC.w;
    float roughnessModified; { const float l = len3(Navg); roughnessModified = sqrt01(roughness * roughness + sat(1.0f - l * l) * positiveRcp(l * (3.0f - l * l))); }     // Filtering::GetModifiedRoughnessFromNormalVariance
    rM1 /= 9.0f; rM2 /= 9.0f;
    const float roughnessSigma = sqrtf(fabsf(rM2 - rM1 * rM1));
    Rng rng; rng.init(uint(x), uint(y), p.frameIndex);
    hitDistForTracking = hitDistForTracking == kInf ? 0.0f : hitDistForTracking;
    const float hitDistNormalization = hitDistanceNormalization(p, viewZ, roughness);
    hitDistForTracking *= p.specPrepassBlurRadius == 0.0f ? hitDistNormalization : 1.0f;
    stHalf(p.trackingCurr, pix, hitDistForTracking);
    // previous position, surface motion
    float3 mv = mk3(0.f);
    if (p.motion) { const uint2 m = p.motion[pix]; mv = mk3(f16tof32(m.x) * rectSizeInv.x, f16tof32(m.x >> 16) * rectSizeInv.y, f16tof32(m.y)); }
    const float2 smbUv = mk2(pixelUv.x + mv.x, pixelUv.y + mv.y);
    const float3 Xprev = rotatePrevInverse(reconstructViewPosition(p.frustumPrev, smbUv, viewZ + mv.z)) + cameraDelta;
    const Bilinear smbBil = bilinearFilter(smbUv, rectSize.x, rectSize.y);
    const int bx = int(smbBil.origin.x), by = int(smbBil.origin.y), ox = bx - 1, oy = by - 1;
    const float pz0[3] = { prevZ(ox + 1, oy), prevZ(ox, oy + 1), prevZ(ox + 1, oy + 1) }, pz1[3] = { prevZ(ox + 2, oy), prevZ(ox + 2, oy + 1), prevZ(ox + 3, oy + 1) };
    const float pz2[3] = { prevZ(ox, oy + 2), prevZ(ox + 1, oy + 2), prevZ(ox + 1, oy + 3) }, pz3[3] = { prevZ(ox + 2, oy + 2), prevZ(ox + 3, oy + 2), prevZ(ox + 2, oy + 3) };
    float3 smbNavg = mk3(0.f);
    {
        const float wz[4] = { pz0[2] < p.denoisingRange ? 1.0f : 0.0f, pz1[1] < p.denoisingRange ? 1.0f : 0.0f, pz2[1] < p.denoisingRange ? 1.0f : 0.0f, pz3[0] < p.denoisingRange ? 1.0f : 0.0f };
        smbNavg = xyz(prevNormalAt(bx, by)) * wz[0] + xyz(prevNormalAt(bx + 1, by)) * wz[1] + xyz(prevNormalAt(bx, by + 1)) * wz[2] + xyz(prevNormalAt(bx + 1, by + 1)) * wz[3];
        const float sum = wz[0] + wz[1] + wz[2] + wz[3]; smbNavg = smbNavg / (sum == 0.0f ? 1.0f : sum);
    }
    auto parallax = [&](float3 Xp, float2 uvZero, const float* M) { const float2 uv = screenUv(M, Xp); const float dx = (uv.x - uvZero.x) * rectSize.x, dy = (uv.y - uvZero.y) * rectSize.y; return sqrtf(dx * dx + dy * dy); };
    const float smbParallax1 = parallax(Xprev + cameraDelta, smbUv, p.worldToClipPrev), smbParallax2 = parallax(Xprev - cameraDelta, pixelUv, p.worldToClip);
    const float smbParallaxMax = fmaxf(smbParallax1, smbParallax2), smbParallaxMin = fminf(smbParallax1, smbParallax2);
    const float pixelSize = pixelRadiusToWorld(p, 1.0f, viewZ), fs = frustumSize(p, viewZ);
    const float disocclusionThreshold = lerpf(p.disocclusionThreshold, p.disocclusionThresholdAlternate, p.disocclusionMix ? float(p.disocclusionMix[pix]) / 255.0f : 0.0f);
    const float thresholdAngle = kAlmostZeroAngle - 0.25f * linearStep(0.25f, 0.0f, smbParallaxMax);
    const float3 V = norm3(-X);
    const float NoV = fabsf(dot3(N, V));
    float thr = fs * sat(disocclusionThreshold / fmaxf(0.05f, lerpf(NoV, 1.0f, sat(smbParallaxMax / 30.0f))));
    thr *= dot3(smbNavg, Navg) > thresholdAngle ? 1.0f : 0.0f;
    const float4 scr = inScreenBilinear(smbBil.origin);
    const float thrQ[4] = { thr * scr.x - kEps, thr * scr.y - kEps, thr * scr.z - kEps, thr * scr.w - kEps };
    const float XvprevZ = p.worldToViewPrev[8] * Xprev.x + p.worldToViewPrev[9] * Xprev.y + p.worldToViewPrev[10] * Xprev.z + p.worldToViewPrev[11];
    float occ0[3], occ1[3], occ2[3], occ3[3];
    {
        const float minMat = fminf(p.minMaterialSpec, p.minMaterialDiff);
        const int t0[3][2] = { { 1, 0 }, { 0, 1 }, { 1, 1 } }, t1[3][2] = { { 2, 0 }, { 2, 1 }, { 3, 1 } }, t2[3][2] = { { 0, 2 }, { 1, 2 }, { 1, 3 } }, t3[3][2] = { { 2, 2 }, { 3, 2 }, { 2, 3 } };
        #pragma unroll
        for (int k = 0; k < 3; k++)
        {
            occ0[k] = (fabsf(pz0[k] - XvprevZ) <= thrQ[0] && compareMaterials(materialID, unpackInternalData(prevInternal(ox + t0[k][0], oy + t0[k][1])).z, minMat)) ? 1.0f : 0.0f;
            occ1[k] = (fabsf(pz1[k] - XvprevZ) <= thrQ[1] && compareMaterials(materialID, unpackInternalData(prevInternal(ox + t1[k][0], oy + t1[k][1])).z, minMat)) ? 1.0f : 0.0f;
            occ2[k] = (fabsf(pz2[k] - XvprevZ) <= thrQ[2] && compareMaterials(materialID, unpackInternalData(prevInternal(ox + t2[k][0], oy + t2[k][1])).z, minMat)) ? 1.0f : 0.0f;
            occ3[k] = (fabsf(pz3[k] - XvprevZ) <= thrQ[3] && compareMaterials(materialID, unpackInternalData(prevInternal(ox + t3[k][0], oy + t3[k][1])).z, minMat)) ? 1.0f : 0.0f;
        }
    }
    const float4 smbOcc = make_float4(occ0[2], occ1[1], occ2[1], occ3[0]);
    const float4 smbW = bilinearCustomWeights(smbBil, smbOcc);
    const bool smbAllowCatRom = (occ0[0] + occ0[1] + occ0[2] + occ1[0] + occ1[1] + occ1[2] + occ2[0] + occ2[1] + occ2[2] + occ3[0] + occ3[1] + occ3[2]) > 11.5f;
    float fbits = smbOcc.x + smbOcc.y * 2.0f + smbOcc.z * 4.0f + smbOcc.w * 8.0f;
    const float3 id00 = unpackInternalData(prevInternal(bx, by)), id10 = unpackInternalData(prevInternal(bx + 1, by)), id01 = unpackInternalData(prevInternal(bx, by + 1)), id11 = unpackInternalData(prevInternal(bx + 1, by + 1));
    float diffAccumSpeed = applyCustomWeights(id00.x, id10.x, id01.x, id11.x, smbW), smbSpecAccumSpeed = applyCustomWeights(id00.y, id10.y, id01.y, id11.y, smbW);
    const float NoVprev = fabsf(dot3(N, norm3(cameraDelta - Xprev)));
    float sizeQuality = (NoVprev + 1e-3f) / (NoV + 1e-3f); sizeQuality = lerpf(0.1f, 1.0f, sat(sizeQuality * sizeQuality));
    const float smbFootprintQuality = sqrt01(applyBilinear(smbOcc.x, smbOcc.y, smbOcc.z, smbOcc.w, smbBil)) * sizeQuality;
    const float2 smbSamplePos = mk2(sat(smbUv.x) * rectSize.x, sat(smbUv.y) * rectSize.y);
    const CatRom smbCat = catRomSetup(smbSamplePos, smbW, smbAllowCatRom);
    const float maxAccum = p.maxAccumulatedFrameNum, maxFast = p.maxFastAccumulatedFrameNum;

    // ---- specular ----
    float specAccumSpeed, curvature, virtualHistoryAmount;
    {
        smbSpecAccumSpeed = fminf(smbSpecAccumSpeed * lerpf(smbFootprintQuality, 1.0f, 1.0f / (1.0f + smbSpecAccumSpeed)), maxAccum);
        const float4 spec = unpackRGBA16F(p.tmp1Spec[pix]);
        {   // curvature along the predicted motion
            const float2 pp = screenUv(p.worldToClipPrev, Xprev + cameraDelta);
            const float dnorm = fmaxf(smbParallax1, 1.0f / 256.0f);
            const float2 deltaUv = mk2((smbUv.x - pp.x) * rectSize.x / dnorm, (smbUv.y - pp.y) * rectSize.y / dnorm);
            auto edgePoint = [&](float ux, float uy) { const float3 xw = viewToWorldRotate(p, reconstructViewPosition(p.frustum, mk2(pixelUv.x + ux, pixelUv.y + uy), 1.0f)); const float3 v = norm3(-xw); return v * (dot3(X, N) / dot3(N, v)); };
            const float3 x10 = edgePoint(rectSizeInv.x, 0.f), x01 = edgePoint(0.f, rectSizeInv.y);
            float wx = fabsf(deltaUv.x) + 1.0f / 256.0f, wy = fabsf(deltaUv.y) + 1.0f / 256.0f; { const float s = wx + wy; wx /= s; wy /= s; }
            float3 xe = x10 * wx + x01 * wy, ne = norm3(xyz(normalAt(x + 1, y)) * wx + xyz(normalAt(x, y + 1)) * wy);
            float deltaUvLenFixed = smbParallaxMin * (1.0f + p.framerateScale * (float(((uint(x) & 3u) + ((uint(y) & 3u) << 2) + p.frameIndex) & 15u) / 16.0f));
            const float2 hi = mk2((floorf((pixelUv.x + deltaUvLenFixed * deltaUv.x * rectSizeInv.x) * rectSize.x) + 0.5f) * rectSizeInv.x, (floorf((pixelUv.y + deltaUvLenFixed * deltaUv.y * rectSizeInv.y) * rectSize.y) + 0.5f) * rectSizeInv.y);
            if (deltaUvLenFixed > 1.0f && inScreen(hi))
            {
                const int hx = clampi(int(floorf(hi.x * rectSize.x)), 0, W - 1), hy = clampi(int(floorf(hi.y * rectSize.y)), 0, H - 1);
                const float zHigh = viewZAt(p, hx, hy);
                if (fabsf(zHigh - viewZ) / fmaxf(zHigh, viewZ) < 0.1f) { ne = xyz(normalAt(hx, hy)); xe = viewToWorldRotate(p, reconstructViewPosition(p.frustum, hi, zHigh)); }
            }
            const float3 edge = xe - X;
            curvature = dot3(ne - N, edge) * positiveRcp(dot3(edge, edge));
        }
        const float3 Xvirt = xVirtual(hitDistForTracking, curvature, X, Xprev, N, V, roughness);
        const float XvirtLength = len3(Xvirt);
        const float2 vmbUv = screenUv(p.worldToClipPrev, Xvirt);
        float2 vmbDelta = mk2(vmbUv.x - smbUv.x, vmbUv.y - smbUv.y);
        const float vmbPixelsTraveled = sqrtf(vmbDelta.x * rectSize.x * vmbDelta.x * rectSize.x + vmbDelta.y * rectSize.y * vmbDelta.y * rectSize.y);
        const Bilinear vmbBil = bilinearFilter(vmbUv, rectSize.x, rectSize.y);
        const int vx = int(vmbBil.origin.x), vy = int(vmbBil.origin.y);
        const int qx4[4] = { 0, 1, 0, 1 }, qy4[4] = { 0, 0, 1, 1 };
        float2 rrw = relaxedRoughnessWeightParams(roughness * roughness, p.roughnessFraction, 0.003f);
        float rwgt[4];
        #pragma unroll
        for (int k = 0; k < 4; k++) { const float r = prevNormalAt(vx + qx4[k], vy + qy4[k]).w; rwgt[k] = lerpf(smoothStep(1.0f, 0.0f, smbParallaxMax), 1.0f, weightWithSigma(r * r, rrw.x, rrw.y, roughnessSigma)); }
        float roughnessConfidence = applyBilinear(rwgt[0], rwgt[1], rwgt[2], rwgt[3], vmbBil);
        auto stochasticPrevNormal = [&](float2 uv) { const Bilinear f = bilinearFilter(uv, rectSize.x, rectSize.y); const float r0 = rng.next(), r1 = rng.next(); return prevNormalAt(int(f.origin.x) + (r0 < f.weights.x ? 1 : 0), int(f.origin.y) + (r1 < f.weights.y ? 1 : 0)); };
        const float4 vmbNR = stochasticPrevNormal(vmbUv); const float3 vmbN = xyz(vmbNR);
        const float Dfactor = specularDominantFactor(NoV, roughness);
        float normalConfidence = 1.0f / (1.0f + 0.5f * Dfactor * sat(len3(N - vmbN) - kNormalEncodingError) * vmbPixelsTraveled);
        if (smbFootprintQuality == 0.0f) smbNavg = vmbN;
        float vmbOcc[4];
        {
            float t = disocclusionThreshold * fs * lerpf(0.25f, 1.0f, NoV);
            t *= dot3(vmbN, N) > thresholdAngle ? 1.0f : 0.0f; t *= dot3(vmbN, smbNavg) > thresholdAngle ? 1.0f : 0.0f;
            const float4 s4 = inScreenBilinear(vmbBil.origin); const float sArr[4] = { s4.x, s4.y, s4.z, s4.w };
            const float3 vmbV = rotatePrevInverse(mk3(vmbUv.x * p.frustumPrev[2] + p.frustumPrev[0], vmbUv.y * p.frustumPrev[3] + p.frustumPrev[1], 1.0f));
            const float NoXcurr = dot3(N, Xprev - cameraDelta);
            #pragma unroll
            for (int k = 0; k < 4; k++)
            {
                const float z = prevZ(vx + qx4[k], vy + qy4[k]);
                const float NoXprev = (N.x * vmbV.x + N.y * vmbV.y) * z + N.z * vmbV.z * z;
                vmbOcc[k] = (fabsf(NoXprev - NoXcurr) <= t * sArr[k] - kEps && rwgt[k] >= 0.5f && compareMaterials(materialID, unpackInternalData(prevInternal(vx + qx4[k], vy + qy4[k])).z, p.minMaterialSpec)) ? 1.0f : 0.0f;
            }
        }
        fbits += vmbOcc[0] * 16.0f + vmbOcc[1] * 32.0f + vmbOcc[2] * 64.0f + vmbOcc[3] * 128.0f;
        const float4 vmbW = bilinearCustomWeights(vmbBil, make_float4(vmbOcc[0], vmbOcc[1], vmbOcc[2], vmbOcc[3]));
        float vmbSpecAccumSpeed = applyCustomWeights(unpackInternalData(prevInternal(vx, vy)).y, unpackInternalData(prevInternal(vx + 1, vy)).y, unpackInternalData(prevInternal(vx, vy + 1)).y, unpackInternalData(prevInternal(vx + 1, vy + 1)).y, vmbW);
        vmbSpecAccumSpeed *= lerpf(sqrt01(applyBilinear(vmbOcc[0], vmbOcc[1], vmbOcc[2], vmbOcc[3], vmbBil)), 1.0f, 1.0f / (1.0f + vmbSpecAccumSpeed));
        const bool vmbAllowCatRom = (vmbOcc[0] + vmbOcc[1] + vmbOcc[2] + vmbOcc[3]) > 3.5f && smbAllowCatRom;
        const float curvatureAngleTan = pixelSize * fabsf(curvature) * fmaxf(vmbPixelsTraveled / fmaxf(NoV, 0.01f), 1.0f) * 2.0f, curvatureAngle = atanf(curvatureAngleTan);
        const float lobeTanHalfAngle = specularLobeTanHalfAngle(roughnessModified, 0.75f / (1.0f + vmbSpecAccumSpeed)), lobeHalfAngle = fmaxf(atanf(lobeTanHalfAngle), kNormalEncodingError);
        auto encodingAwareNormalWeight = [&](float3 a, float3 b, float curvAngle) { return smoothStep01(1.0f - (acosApprox(dot3(a, b)) - curvAngle - kNormalEncodingError) / lobeHalfAngle); };
        normalConfidence = fminf(normalConfidence, lerpf(smoothStep(1.0f, 0.0f, vmbPixelsTraveled), 1.0f, encodingAwareNormalWeight(N, vmbN, curvatureAngle)));
        virtualHistoryAmount = smoothStep(0.05f, 0.95f, Dfactor) * normalConfidence;
        float parallaxConfidence;
        {
            const float hitDistPrev = sampleBilinear1(p.trackingPrev, W, H, mk2(vmbUv.x * rectSize.x, vmbUv.y * rectSize.y));
            const float2 uvPrev = screenUv(p.worldToClipPrev, xVirtual(hitDistPrev, curvature, X, Xprev, N, V, roughness));
            const float r = fmaxf((lobeTanHalfAngle + curvatureAngleTan) * fminf(hitDistForTracking, hitDistPrev) / pixelRadiusToWorld(p, 1.0f, XvirtLength), 0.1f);
            const float dx = (uvPrev.x - vmbUv.x) * rectSize.x, dy = (uvPrev.y - vmbUv.y) * rectSize.y;
            parallaxConfidence = linearStep(r, 0.0f, sqrtf(dx * dx + dy * dy));
        }
        {   // prev-prev test along the virtual motion (1 iteration)
            const float step = fminf(vmbPixelsTraveled * p.framerateScale, 2.0f) + vmbPixelsTraveled;
            const float inv = rsqrtf(vmbDelta.x * vmbDelta.x + vmbDelta.y * vmbDelta.y);
            const float2 uvPrev = mk2(vmbUv.x + vmbDelta.x * inv / rectSize.x * step, vmbUv.y + vmbDelta.y * inv / rectSize.y * step);
            rrw = relaxedRoughnessWeightParams(vmbNR.w * vmbNR.w, p.roughnessFraction, 0.003f);
            if (isfinite(uvPrev.x) && isfinite(uvPrev.y) && inScreen(uvPrev))
            {
                const float4 nrPrev = stochasticPrevNormal(uvPrev);
                const float wn = lerpf(1.0f, encodingAwareNormalWeight(vmbN, xyz(nrPrev), curvatureAngle * (1.0f + step)), sat(step)), wr = lerpf(1.0f, weightWithSigma(nrPrev.w * nrPrev.w, rrw.x, rrw.y, roughnessSigma), sat(step));
                normalConfidence = fminf(normalConfidence, wn); roughnessConfidence = fminf(roughnessConfidence, wr);
            }
        }
        const float confidenceForSmbRelaxation = normalConfidence * roughnessConfidence, virtualConfidence = confidenceForSmbRelaxation * parallaxConfidence;
        virtualHistoryAmount *= roughnessConfidence;
        float4 smbHist = catRomSample4(smbCat, p.specHistory, W, H); const float smbFastHist = footprintSample1(smbCat.centerPos, smbW, p.specFast, W, H);
        float surfaceConfidence;
        {
            const float a = atanf(smbParallaxMax * pixelSize / len3(X)), nl = 1.0f / (1.0f + smbSpecAccumSpeed);
            const float hd = lerpf(smbHist.w, spec.w, nl) * hitDistNormalization;
            const float tana0 = specularLobeTanHalfAngle(roughnessModified, 0.75f) * lerpf(NoV, 1.0f, roughnessModified) * nl / (sat(hd / fs) + kEps);
            surfaceConfidence = pow01(linearStep(fmaxf(atanf(tana0), kNormalEncodingError), 0.0f, a), 4.0f);
        }
        float2 maxResponsive;
        {
            const float responsiveFactor = smoothStep01((roughness + kEps) / (p.responsiveAccumulationRoughnessThreshold + kEps)), smc = specMagicCurve(roughnessModified);
            const float fa = lerpf(smc, 1.0f, responsiveFactor), pw = lerpf(32.0f, 1.0f, smc) * (1.0f - responsiveFactor);
            maxResponsive = mk2(fmaxf(maxAccum * fa * pow01(dot3(N, norm3(smbNavg)), pw), p.historyFixFrameNum), fmaxf(maxAccum * fa * pow01(dot3(N, vmbN), pw), p.historyFixFrameNum));
        }
        const float smbMaxFrameNum = fminf(maxAccum * surfaceConfidence, maxResponsive.x);
        const float smbBoosted = fminf(smbSpecAccumSpeed, fmaxf(smbMaxFrameNum, p.historyFixFrameNum * (1.0f - confidenceForSmbRelaxation)));
        smbSpecAccumSpeed = fminf(smbSpecAccumSpeed, smbMaxFrameNum); vmbSpecAccumSpeed = fminf(vmbSpecAccumSpeed, fminf(maxAccum * virtualConfidence, maxResponsive.y));
        const float amountUnbiased = virtualHistoryAmount;
        virtualHistoryAmount = sat(virtualHistoryAmount * (1.0f + (vmbSpecAccumSpeed - smbSpecAccumSpeed) / ((vmbSpecAccumSpeed > smbSpecAccumSpeed ? 8.0f : 0.5f) * fmaxf(vmbSpecAccumSpeed, smbSpecAccumSpeed) + 1.0f)));
        const CatRom vmbCat = catRomSetup(mk2(sat(vmbUv.x) * rectSize.x, sat(vmbUv.y) * rectSize.y), vmbW, vmbAllowCatRom);
        float4 vmbHist = catRomSample4(vmbCat, p.specHistory, W, H); const float vmbFastHist = footprintSample1(vmbCat.centerPos, vmbW, p.specFast, W, H);
        smbHist = clampNegativeToZero(smbHist); vmbHist = clampNegativeToZero(vmbHist);
        const float4 smbSpec = mixHistoryAndCurrent(p, smbHist, spec, 1.0f / (1.0f + smbSpecAccumSpeed), roughnessModified), vmbSpec = mixHistoryAndCurrent(p, vmbHist, spec, 1.0f / (1.0f + vmbSpecAccumSpeed), roughnessModified);
        float4 result = smbSpec * (1.0f - virtualHistoryAmount) + vmbSpec * virtualHistoryAmount;
        specAccumSpeed = lerpf(smbBoosted, vmbSpecAccumSpeed, virtualHistoryAmount);
        const float histLuma = smbHist.x * (1.0f - virtualHistoryAmount) + vmbHist.x * virtualHistoryAmount;
        const float maxRelative = p.fireflySuppressorMinRelativeScale + 38.0f / (specAccumSpeed + 1.0f);
        float antifirefly = specAccumSpeed * p.maxBlurRadius * 0.1f; antifirefly /= 1.0f + antifirefly;
        result = changeLuma(result, lerpf(result.x, fminf(result.x, histLuma * maxRelative), antifirefly));
        p.tmp2Spec[pix] = packRGBA16F(result);
        const float smbFast = lerpf(smbFastHist, spec.x, fmaxf(1.0f - surfaceConfidence, 1.0f / (1.0f + fminf(smbSpecAccumSpeed, maxFast)))), vmbFast = lerpf(vmbFastHist, spec.x, fmaxf(1.0f - virtualConfidence, 1.0f / (1.0f + fminf(vmbSpecAccumSpeed, maxFast))));
        float fast = lerpf(smbFast, vmbFast, amountUnbiased);
        fast = lerpf(fast, fminf(fast, histLuma * maxRelative * 4.0f), antifirefly);
        stHalf(p.specFastTransient, pix, fast);
    }
    p.data2[pix] = uint(fbits + 0.5f) | (uint(sat(virtualHistoryAmount) * 127.0f + 0.5f) << 8) | (smbAllowCatRom ? (1u << 15) : 0u) | (f32tof16(curvature) << 16);
    // ---- diffuse ----
    {
        diffAccumSpeed = fminf(diffAccumSpeed * lerpf(smbFootprintQuality, 1.0f, 1.0f / (1.0f + diffAccumSpeed)), maxAccum);
        const float4 diff = unpackRGBA16F(p.tmp1Diff[pix]);
        const float4 hist = clampNegativeToZero(catRomSample4(smbCat, p.diffHistory, W, H)); const float fastHist = footprintSample1(smbCat.centerPos, smbW, p.diffFast, W, H);
        float4 result = mixHistoryAndCurrent(p, hist, diff, 1.0f / (1.0f + diffAccumSpeed), 1.0f);
        const float maxRelative = p.fireflySuppressorMinRelativeScale + 38.0f / (diffAccumSpeed + 1.0f);
        float antifirefly = diffAccumSpeed * p.maxBlurRadius * 0.1f; antifirefly /= 1.0f + antifirefly;
        result = changeLuma(result, lerpf(result.x, fminf(result.x, hist.x * maxRelative), antifirefly));
        p.tmp2Diff[pix] = packRGBA16F(result);
        float fast = lerpf(fastHist, diff.x, 1.0f / (1.0f + fminf(diffAccumSpeed, maxFast)));
        fast = lerpf(fast, fminf(fast, hist.x * maxRelative * 4.0f), antifirefly);
        stHalf(p.diffFastTransient, pix, fast);
    }
    p.data1[pix] = make_uchar2((unsigned char)(sat(diffAccumSpeed / 63.0f) * 255.0f + 0.5f), (unsigned char)(sat(specAccumSpeed / 63.0f) * 255.0f + 0.5f));
}

// ---- HistoryFix: tmp2 + transient fast -> tmp1, permanent fast ----------------------------------------------------------------------------------------------------------------
PT_HD void historyFixPixel(const Params& p, const int x, const int y)
{
    RB_PIXEL_PROLOGUE;
    float materialID; const float4 nr = unpackNormalRoughness(p.normalRoughness[pix], materialID);
    const float3 N = xyz(nr), Nv = worldToViewRotate(p, N); const float roughness = nr.w;
    const float fs = frustumSize(p, viewZ);
    const float3 Xv = reconstructViewPosition(p.frustum, pixelUv, viewZ);
    auto frames = [&](int qx, int qy) { const uchar2 q = p.data1[size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)]; return mk2(float(q.x) / 255.0f * 63.0f, float(q.y) / 255.0f * 63.0f); };
    const float2 frameNum = frames(x, y);
    float2 stride;
    {
        float ax = frameNum.x, ay = frameNum.y, sx = 1.0f, sy = 1.0f; const float inv = 1.0f / (p.historyFixFrameNum + kEps);
        for (int i = -1; i <= 1; i++) for (int j = -1; j <= 1; j++)
        {
            if (i == 0 && j == 0) continue;
            const float2 f = frames(x + i, y + j); const float wx = f.x >= frameNum.x ? 1.0f : 0.0f, wy = f.y >= frameNum.y ? 1.0f : 0.0f;
            ax += sat(f.x * inv) * wx; ay += sat(f.y * inv) * wy; sx += wx; sy += wy;
        }
        stride = mk2(p.historyFixBasePixelStride / (2.0f + ax / sx * p.historyFixFrameNum) * (frameNum.x < p.historyFixFrameNum ? 1.0f : 0.0f), p.historyFixBasePixelStride / (2.0f + ay / sy * p.historyFixFrameNum) * (frameNum.y < p.historyFixFrameNum ? 1.0f : 0.0f));
    }
    #pragma unroll 1
    for (int channel = 0; channel < 2; channel++)
    {
        const bool isSpec = channel == 1;
        const uint2* src = isSpec ? p.tmp2Spec : p.tmp2Diff; const unsigned short* fast = isSpec ? p.specFastTransient : p.diffFastTransient;
        float4 v = unpackRGBA16F(src[pix]);
        const float smc = specMagicCurve(roughness), fn = isSpec ? frameNum.y : frameNum.x, r = isSpec ? roughness : 1.0f;
        const float st = floorf(isSpec ? stride.y * lerpf(0.5f, 1.0f, smc) : stride.x);
        if (st != 0.0f)
        {
            const int sti = int(st + 0.5f); const float nl = 1.0f / (1.0f + fn);
            const float normalW = normalWeightParam(nl, p.lobeAngleFraction, r);
            const float2 gw = geometryWeightParams(p, fs, Xv, Nv), rw = relaxedRoughnessWeightParams(roughness * roughness, sqrtf(p.roughnessFraction), 0.01f);
            const float hitDistScale = hitDistanceNormalization(p, viewZ, r), hitDist = v.w * hitDistScale;
            const float2 hw = hitDistanceWeightParams(sat(hitDist / fs), nl, r);
            float sum = 1.0f + fn; v = v * sum;
            for (int j = -2; j <= 2; j++) for (int i = -2; i <= 2; i++)
            {
                if ((i == 0 && j == 0) || (abs(i) + abs(j) == 4)) continue;
                const float2 uv = mk2(pixelUv.x + float(i) * st * rectSizeInv.x, pixelUv.y + float(j) * st * rectSizeInv.y);
                const int qx = clampi(x + i * sti, 0, W - 1), qy = clampi(y + j * sti, 0, H - 1); const size_t q = size_t(qy) * W + qx;
                float ms; const float4 Ns = unpackNormalRoughness(p.normalRoughness[q], ms);
                float w = inScreen(uv) ? 1.0f : 0.0f;
                w *= weight(dot3(Nv, reconstructViewPosition(p.frustum, uv, viewZAt(p, qx, qy))), gw.x, gw.y);
                w *= compareMaterials(materialID, ms, isSpec ? p.minMaterialSpec : p.minMaterialDiff) ? 1.0f : 0.0f;
                w *= exponentialWeight(acosApprox(dot3(xyz(Ns), N)), normalW, 0.0f);
                if (isSpec) w *= exponentialWeight(Ns.w * Ns.w, rw.x, rw.y);
                const float2 fq = frames(qx, qy); w *= 1.0f + (isSpec ? fq.y : fq.x);
                float4 sv = unpackRGBA16F(src[q]); if (w == 0.0f) sv = make_float4(0, 0, 0, 0);
                const float hs = sv.w * hitDistScale;
                w *= exponentialWeight(sat(hs / fs), hw.x, hw.y);
                if (isSpec) { const float d = fabsf(hitDist - hs) / (fmaxf(hitDist, hs) + 0.001f), b = linearStep(0.03f, 0.05f, roughness); w *= smoothStep(0.2f + b, 0.05f + b, d); }
                sum += w; v = v + sv * w;
            }
            v = v * positiveRcp(sum);
        }
        auto fastAt = [&](int qx, int qy) { return ldHalf(fast, size_t(clampi(qy, 0, H - 1)) * W + clampi(qx, 0, W - 1)); };
        float center = fastAt(x, y), m1 = center, m2 = center * center;
        float f = sat(fn / (p.historyFixFrameNum + kEps)); if (isSpec) f = lerpf(1.0f, f, smc);
        stHalf(isSpec ? p.specFast : p.diffFast, pix, lerpf(v.x, center, f));
        for (int j = -2; j <= 2; j++) for (int i = -2; i <= 2; i++) { if (i == 0 && j == 0) continue; const float d = fastAt(x + i, y + j); m1 += d; m2 += d * d; }
        float luma = v.x;
        if (p.antiFirefly)
        {
            float a1 = 0.f, a2 = 0.f;
            for (int j = -4; j <= 4; j++) for (int i = -4; i <= 4; i++) { if (abs(i) <= 1 && abs(j) <= 1) continue; const float d = fastAt(x + i, y + j); a1 += d; a2 += d * d; }
            a1 /= 72.0f; a2 /= 72.0f;
            const float sigma = sqrtf(fabsf(a2 - a1 * a1)) * 2.0f;
            luma = clampf(luma, a1 - sigma, a1 + sigma);
        }
        m1 /= 25.0f; m2 /= 25.0f;
        const float sigma = sqrtf(fabsf(m2 - m1 * m1)) * 2.0f;
        luma = lerpf(clampf(luma, m1 - sigma, m1 + sigma), luma, 1.0f / (1.0f + (p.maxFastAccumulatedFrameNum < p.maxAccumulatedFrameNum ? 1.0f : 0.0f) * fn * 2.0f));
        (isSpec ? p.tmp1Spec : p.tmp1Diff)[pix] = packRGBA16F(changeLuma(v, luma));
    }
}

// ---- TemporalStabilization: history (post-blurred) + stabilised luminance history -> outputs, internal data --------------------------------------------------------------------
PT_HD void temporalStabilizationPixel(const Params& p, const int x, const int y)
{
    RB_PIXEL_PROLOGUE_SKY(p.diffLumaCurr[pix] = p.diffLumaPrev[pix]; p.specLumaCurr[pix] = p.specLumaPrev[pix]; p.outDiff[pix] = p.diffHistory[pix]; p.outSpec[pix] = p.specHistory[pix]);
    const float2 rectSize = mk2(float(W), float(H));
    const float3 Xv = reconstructViewPosition(p.frustum, pixelUv, viewZ), X = viewToWorldRotate(p, Xv);
    const float3 cameraDelta = mk3(p.cameraDelta[0], p.cameraDelta[1], p.cameraDelta[2]);
    float3 mv = mk3(0.f);
    if (p.motion) { const uint2 m = p.motion[pix]; mv = mk3(f16tof32(m.x) * rectSizeInv.x, f16tof32(m.x >> 16) * rectSizeInv.y, f16tof32(m.y)); }
    const float2 smbUv = mk2(pixelUv.x + mv.x, pixelUv.y + mv.y);
    float3 Xprev; { const float3 v = reconstructViewPosition(p.frustumPrev, smbUv, viewZ + mv.z); const float* t = p.worldToViewPrev; Xprev = mk3(t[0] * v.x + t[4] * v.y + t[8] * v.z, t[1] * v.x + t[5] * v.y + t[9] * v.z, t[2] * v.x + t[6] * v.y + t[10] * v.z) + cameraDelta; }
    float materialID; const float4 nr = unpackNormalRoughness(p.normalRoughness[pix], materialID);
    const float3 N = xyz(nr); const float roughness = nr.w;
    float2 d1; { const uchar2 q = p.data1[pix]; d1 = mk2(float(q.x) / 255.0f * 63.0f, float(q.y) / 255.0f * 63.0f); }
    const uint p2 = p.data2[pix], bits = p2 & 0xFFu; const bool smbAllowCatRom = (p2 & (1u << 15)) != 0;
    const float virtualHistoryAmount = float((p2 >> 8) & 127u) / 127.0f, curvature = f16tof32(p2 >> 16);
    const Bilinear smbBil = bilinearFilter(smbUv, rectSize.x, rectSize.y);
    const float4 smbOcc = make_float4((bits & 1u) ? 1.f : 0.f, (bits & 2u) ? 1.f : 0.f, (bits & 4u) ? 1.f : 0.f, (bits & 8u) ? 1.f : 0.f);
    const float4 smbW = bilinearCustomWeights(smbBil, smbOcc);
    const float smbFootprintQuality = sqrt01(applyBilinear(smbOcc.x, smbOcc.y, smbOcc.z, smbOcc.w, smbBil));
    const CatRom smbCat = catRomSetup(mk2(sat(smbUv.x) * rectSize.x, sat(smbUv.y) * rectSize.y), smbW, smbAllowCatRom);
    auto antilag = [&](float history, float avg, float sigma, float accumSpeed) {
        const float s = sigma * p.antilagSigmaScale, magic = p.antilagSensitivity * p.framerateScale * p.framerateScale;
        const float hc = clampf(history, avg - s, avg + s);
        return 1.0f / (1.0f + fabsf(history - hc) / (fmaxf(history, hc) + kEps) * accumSpeed / magic); };
    auto moments = [&](const uint2* img, float& luma, float& m1, float& sigma) {
        luma = f16tof32(img[pix].x); float a = luma, b = luma * luma, mn = kInf, mx = -kInf;
        for (int j = -1; j <= 1; j++) for (int i = -1; i <= 1; i++) { if (i == 0 && j == 0) continue; const float d = f16tof32(img[size_t(clampi(y + j, 0, H - 1)) * W + clampi(x + i, 0, W - 1)].x); a += d; b += d * d; mn = fminf(mn, d); mx = fmaxf(mx, d); }
        m1 = a / 9.0f; sigma = sqrtf(fabsf(b / 9.0f - m1 * m1));
        if (p.maxBlurRadius != 0.0f) luma = clampf(luma, mn, mx); };
    {   // diffuse
        float luma, m1, sigma; moments(p.diffHistory, luma, m1, sigma);
        float hist = fmaxf(catRomSample1(smbCat, p.diffLumaPrev, W, H), 0.0f);
        const float al = antilag(hist, m1, sigma, smbFootprintQuality * d1.x);
        float wgt = smbFootprintQuality * (d1.x / (1.0f + d1.x)); const float clampScale = 1.0f + 3.0f * p.framerateScale * wgt;
        wgt *= al;
        hist = clampf(hist, m1 - sigma * clampScale, m1 + sigma * clampScale);
        const float stabilized = lerpf(luma, hist, fminf(wgt, p.stabilizationStrength));
        p.outDiff[pix] = packRGBA16F(changeLuma(unpackRGBA16F(p.diffHistory[pix]), stabilized)); stHalf(p.diffLumaCurr, pix, stabilized);
        d1.x += 1.0f; d1.x = lerpf(fminf(d1.x, p.historyFixFrameNum), d1.x, al);
    }
    {   // specular
        float luma, m1, sigma; moments(p.specHistory, luma, m1, sigma);
        const float4 spec = unpackRGBA16F(p.specHistory[pix]);
        float hitDistForTracking = spec.w * hitDistanceNormalization(p, viewZ, roughness);
        if (p.specPrepassBlurRadius != 0.0f) hitDistForTracking = fminf(hitDistForTracking, ldHalf(p.trackingCurr, pix));
        const float3 V = norm3(-X);
        const float2 vmbUv = screenUv(p.worldToClipPrev, xVirtual(hitDistForTracking, curvature, X, Xprev, N, V, roughness));
        const float smbHist = fmaxf(catRomSample1(smbCat, p.specLumaPrev, W, H), 0.0f);
        const Bilinear vmbBil = bilinearFilter(vmbUv, rectSize.x, rectSize.y);
        const float4 vmbOcc = make_float4((bits & 16u) ? 1.f : 0.f, (bits & 32u) ? 1.f : 0.f, (bits & 64u) ? 1.f : 0.f, (bits & 128u) ? 1.f : 0.f);
        const bool vmbAllowCatRom = (vmbOcc.x + vmbOcc.y + vmbOcc.z + vmbOcc.w) > 3.5f && smbAllowCatRom;
        const float vmbFootprintQuality = sqrt01(applyBilinear(vmbOcc.x, vmbOcc.y, vmbOcc.z, vmbOcc.w, vmbBil));
        const CatRom vmbCat = catRomSetup(mk2(sat(vmbUv.x) * rectSize.x, sat(vmbUv.y) * rectSize.y), bilinearCustomWeights(vmbBil, vmbOcc), vmbAllowCatRom);
        const float vmbHist = fmaxf(catRomSample1(vmbCat, p.specLumaPrev, W, H), 0.0f);
        float hist = lerpf(smbHist, vmbHist, virtualHistoryAmount);
        const float footprintQuality = lerpf(smbFootprintQuality, vmbFootprintQuality, virtualHistoryAmount);
        const float al = antilag(hist, m1, sigma, footprintQuality * d1.y);
        float wgt = footprintQuality * (d1.y / (1.0f + d1.y)); const float clampScale = 1.0f + 3.0f * p.framerateScale * wgt;
        wgt *= al;
        wgt *= lerpf(specMagicCurve(roughness), 1.0f, 0.5f + smoothStep01((roughness + kEps) / (p.responsiveAccumulationRoughnessThreshold + kEps)) * 0.5f);
        hist = clampf(hist, m1 - sigma * clampScale, m1 + sigma * clampScale);
        const float stabilized = lerpf(luma, hist, fminf(wgt, p.stabilizationStrength));
        p.outSpec[pix] = packRGBA16F(changeLuma(spec, stabilized)); stHalf(p.specLumaCurr, pix, stabilized);
        d1.y += 1.0f; d1.y = lerpf(fminf(d1.y, p.historyFixFrameNum), d1.y, al);
    }
    p.prevInternalData[pix] = (unsigned short)packInternalData(d1.x, d1.y, materialID);
}


} } // namespace pt::rb
