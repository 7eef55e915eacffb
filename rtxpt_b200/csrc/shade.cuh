// shade.cuh — what the reference's closest-hit / miss shaders do for one path vertex, as device functions of the shade kernel.
//   surface load:   Bridge::loadSurface + getGeometryFromHit + sampleGeometryMaterialRTXPT + EvaluateSceneMaterialRTXPT
//                   (Rtxpt/Shaders/PathTracerBridgeDonut.hlsli:152-256, :311-428, :612-853), computeTangentSpace / adjustShadingNormal
//                   (PathTracer/Scene/Material/ShadingUtils.hlsli:110-166), ray-cone LOD (Rendering/Materials/TexLODHelpers.hlsli:41-161,
//                   Scene/Material/TextureSampler.hlsli ExplicitRayConesLodTextureSampler)
//   miss:           PathTracer::HandleMiss (PathTracer/PathTracer.hlsli:407-503)
//   hit:            PathTracer::HandleHit (:505-762), GenerateScatterRay (:217-380), HandleRussianRoulette (:182-208),
//                   HandleNestedDielectrics (PathTracerNestedDielectrics.hlsli:48-131), InteriorList (InteriorList.hlsli)
//   NEE:            HandleNEE / GenerateLightSample / ProcessLightSample (PathTracerNEE.hlsli:41-346) with the global proxy sampler
//                   (Lighting/LightSampler.hlsli:109-117, :282-328), TriangleLight / EnvironmentQuadLight
//                   (Lighting/PolymorphicLight.hlsli:395-520, :560-640)
// The NEE visibility ray is not traced here: the shade kernel emits a shadow record carrying the radiance "if visible" and the
// shadow kernel adds it to L — same arithmetic and order as ProcessLightSample followed by AccumulatePathRadiance.  With NEEFullSamples > 1
// (MULTI) every valid light sample gets its own shadow record and parks its fp32 result in the vertex's NEE block (wavefront.cuh); the shadow
// kernel marks the visible ones and k_nee_resolve sums them in sample order before the one AccumulatePathRadiance.
// Light-vs-BSDF MIS comes in RTXPT's two kinds (RTXPT_USE_APPROXIMATE_MIS): full (ComputeLightVsBSDF_MIS_ForLight / ForBSDF, LightSampler.hlsli:282-331) and, with AMIS,
// approximate (the _Approx pair, :271-280), a compile-time choice as in the reference; RtxptPathTracerConstants::useApproximateMIS selects the kernel.
#pragma once
#include "wavefront.cuh"
#include "bsdf.cuh"
#include "stf.cuh"
#include "debug_views.cuh"

namespace pt {

// ---- textures -----------------------------------------------------------------------------------------------------------------
PT_DEVICE float4 sampleMaterialTexture(const SceneView& sc, uint textureIndexAndInfo, float lodNoDims, float2 uv)
{
    const uint textureIndex = textureIndexAndInfo & 0xFFFF, baseLOD = textureIndexAndInfo >> 24, mipLevels = (textureIndexAndInfo >> 16) & 0xFF;
    float lambda = 0.5f * float(baseLOD) + lodNoDims;
    lambda = fminf(lambda, fmaxf(float(mipLevels) - 5.0f, 0.0f));
    return tex2DLod<float4>(sc.textures[textureIndex], uv.x, uv.y, lambda);
}
// Stochastic texture filtering (rtxpt_b200_set_texture_filtering): ExplicitRayConesLodTextureSampler's lambda, then STF_SamplerState::Texture2DSampleLevel - one texel of one integer
// level, fetched at its centre through the point-filtered object over the same mip arrays, so that the texture unit returns the texel itself.  `stf` arrives by value: the bridge hands
// the sampler to every fetch as a copy (sampleTexture's `const ActiveTextureSampler` parameter, BridgeDonut:269-278), so each fetch of a vertex starts from the vertex's state.
PT_DEVICE float4 sampleMaterialTextureStf(const LaunchParams& p, uint textureIndexAndInfo, float lodNoDims, float2 uv, StfState stf)
{
    const uint textureIndex = textureIndexAndInfo & 0xFFFF, baseLOD = textureIndexAndInfo >> 24, mipLevels = (textureIndexAndInfo >> 16) & 0xFF;
    float lambda = 0.5f * float(baseLOD) + lodNoDims;
    lambda = fminf(lambda, fmaxf(float(mipLevels) - 5.0f, 0.0f));
    const uint4 dims = p.stf.textureDims[textureIndex];             // Texture2D::GetDimensions(0, ...): width, height, number of levels
    const StfSamplePos pos = stfTexture2DSamplePos(stf, dims.x, dims.y, dims.z, uv, lambda);
    return tex2DLod<float4>(p.stf.pointTextures[textureIndex], pos.uv.x, pos.uv.y, float(pos.lod));
}
PT_DEVICE float safeLog2(float x) { return log2f(clampf(x, kFltMin, kFltMax)); }

// D3D cube face selection; the cube is bound as a 6-layer 2D texture so that face/uv selection is this code on both sides of the parity test
PT_DEVICE float3 sampleEnvCube(const SceneView& sc, float3 v, float lod)
{
    if (sc.envFaceSize == 0) return mk3(0.f);
    const float ax = fabsf(v.x), ay = fabsf(v.y), az = fabsf(v.z);
    float m, s, t; int face;
    if (ax >= ay && ax >= az) { m = ax; if (v.x >= 0) { face = 0; s = -v.z; t = -v.y; } else { face = 1; s = v.z; t = -v.y; } }
    else if (ay >= az)        { m = ay; if (v.y >= 0) { face = 2; s = v.x; t = v.z; }  else { face = 3; s = v.x; t = -v.z; } }
    else                      { m = az; if (v.z >= 0) { face = 4; s = v.x; t = -v.y; } else { face = 5; s = -v.x; t = -v.y; } }
    const float level = clampf(floorf(lod + 0.5f), 0.0f, float(sc.envMipLevels - 1));
    const float4 c = tex2DLayeredLod<float4>(sc.envCube, (s / m + 1.0f) * 0.5f, (t / m + 1.0f) * 0.5f, face, level);
    return mk3(c.x, c.y, c.z);
}
#ifdef PT_HOST_EMU     // tests/emu/shade_host_emu.cu (test infrastructure): the environment cube and the triangle gather are what the golden vectors' stub bridge supplies as data
__host__ __device__ float3 emuEnvCube(float3 localDir, float lod);
#endif
PT_DEVICE float3 envEvalLocal(const LaunchParams& p, float3 localDir, float lod)     // EnvMap::EvalLocal, Lighting/EnvMap.hlsli:84-87
{
#ifdef PT_HOST_EMU
    return emuEnvCube(localDir, lod) * mk3(p.c.envMap.ColorMultiplier[0], p.c.envMap.ColorMultiplier[1], p.c.envMap.ColorMultiplier[2]);
#endif
    return sampleEnvCube(p.scene, localDir, lod) * mk3(p.c.envMap.ColorMultiplier[0], p.c.envMap.ColorMultiplier[1], p.c.envMap.ColorMultiplier[2]);
}

// ---- lights ----------------------------------------------------------------------------------------------------------------------
constexpr uint kLightTypeSphere = 0, kLightTypeTriangle = 1, kLightTypeEnvQuad = 5;
constexpr uint kLightShapingEnableBit = 1u << 28, kLightShapingUseMinFalloff = 1u << 30;
constexpr float kDistantLightDistance = 100000.0f;
constexpr uint kEnvLookupDim = 1024;
constexpr uint kInvalidLight = 0xFFFFFFFFu;

PT_DEVICE uint lightType(const LightInfo& li) { return (li.colorTypeAndFlags >> 24) & 0xf; }
PT_DEVICE float3 unpackLightRadiance(const LightInfo& li)           // PolymorphicLight::UnpackColor/UnpackRadiance
{
    const uint lr = li.logRadiance & 0xffff;
    const float radiance = (lr == 0) ? 0.f : exp2f((float(lr - 1) / 65534.0f) * 48.0f + -8.0f);
    return mk3(unpackUnorm8(li.colorTypeAndFlags), unpackUnorm8(li.colorTypeAndFlags >> 8), unpackUnorm8(li.colorTypeAndFlags >> 16)) * radiance;
}

// evaluateLightShaping (LightShaping.hlsli:26-95): spot falloff of a shaped light towards `surfacePos`, 1 for unshaped lights
PT_DEVICE float lightShaping(const LightInfo& li, const SceneView& sc, uint lightIndex, float3 surfacePos, float3 lightSamplePos)
{
    if (!(li.colorTypeAndFlags & kLightShapingEnableBit)) return 1.0f;
    const uint4 ex = sc.lightsEx[lightIndex - 5368u];
    const float3 axis = octUnorm32ToDir(ex.y);
    const float cosCone = f16tof32(ex.z), softness = f16tof32(ex.z >> 16);
    const float minFalloff = (li.colorTypeAndFlags & kLightShapingUseMinFalloff) ? 0.0001f : 0.0f;
    const float cosT = dot3(axis, norm3(surfacePos - lightSamplePos));
    const float t = sat((cosT - cosCone) / ((cosCone + softness) - cosCone));
    const float falloff = fmaxf(minFalloff, t * t * (3.0f - 2.0f * t));
    return falloff <= 0 ? 0.0f : falloff;
}
// SphereLight::CalcSample + evaluateLightShaping (PolymorphicLight.hlsli:107-181, :669-673; LightShaping.hlsli:26-95)
PT_DEVICE void sampleSphereLight(const LightInfo& li, const SceneView& sc, uint lightIndex, float u0, float u1, float3 viewer, float3& outPos, float3& outRadiance, float& outSolidPdf)
{
    const float3 center = mk3(li.cx, li.cy, li.cz);
    const float radius = f16tof32(li.scalars);
    const float3 lightVector = center - viewer;
    const float d2 = dot3(lightVector, lightVector), r2 = radius * radius;
    if (d2 < r2) { outPos = center; outRadiance = mk3(0.f); outSolidPdf = 1.0f; return; }      // viewer inside: single-sided emitter
    const float dc = sqrtf(d2);
    const float cosThetaMax = sqrtf(fmaxf(0.0f, 1.0f - r2 / d2));
    const float phi = 2.0f * kPi * u0;
    const float cosTheta = cosThetaMax + (1.0f - cosThetaMax) * u1;
    const float sinTheta = sqrtf(fmaxf(0.0f, 1.0f - cosTheta * cosTheta));
    const float ds = dc * cosTheta - sqrtf(fmaxf(1e-10f, r2 - d2 * (sinTheta * sinTheta)));
    const float cosAlpha = (d2 + r2 - ds * ds) / (2.0f * dc * radius);
    const float sinAlpha = sqrtf(fmaxf(0.0f, 1.0f - cosAlpha * cosAlpha));
    const float3 n = norm3(lightVector);
    const float sign = (n.z >= 0) ? 1.0f : -1.0f;                   // BranchlessONB (Utils/Geometry.hlsli:17-24)
    const float a = -1.0f / (sign + n.z), b = n.x * n.y * a;
    const float3 T = mk3(1.0f + sign * n.x * n.x * a, sign * b, -sign * n.x), B = mk3(b, sign + n.y * n.y * a, -n.y);
    const float sinPhi = sinf(phi), cosPhi = cosf(phi);
    const float3 radiusVector = (-T) * (sinAlpha * cosPhi) + (-B) * (sinAlpha * sinPhi) + (-n) * cosAlpha;
    outPos = center + radiusVector * radius;
    outSolidPdf = 1.0f / (2.0f * kPi * (1.0f - cosThetaMax));
    outRadiance = unpackLightRadiance(li) * lightShaping(li, sc, lightIndex, viewer, outPos);
}
struct TriLight
{
    float3 base, e1, e2, radiance, normal; float area;
    PT_DEVICE void decode(const LightInfo& li)                      // TriangleLight::Create, PolymorphicLight.hlsli:478-503
    {
        e1 = mk3(f16tof32(li.direction1), f16tof32(li.direction2), f16tof32(li.scalars));
        e2 = mk3(f16tof32(li.direction1 >> 16), f16tof32(li.direction2 >> 16), f16tof32(li.scalars >> 16));
        base = mk3(li.cx, li.cy, li.cz) - ((e1 + e2) / 3.0f);
        radiance = unpackLightRadiance(li);
        const float3 n = cross3(e1, e2);
        const float len = len3(n);
        if (len > 0.0f) { area = 0.5f * len; normal = n / len; } else { area = 0.0f; normal = mk3(0.f); }
    }
    PT_DEVICE float solidAnglePdfForMIS(float3 viewer, float3 samplePos) const      // PolymorphicLight.hlsli:443-454
    {
        const float3 toLight = samplePos - viewer;
        const float dist = sqrtf(fmaxf(2e-9f, dot3(toLight, toLight)));
        const float cosTheta = dot3(normal, -(toLight / dist));
        return fminf(1e10f, pdfAreaToSolidAngle(fmaxf(2e-9f, 1.0f / area), dist, cosTheta));
    }
};
PT_DEVICE float globalLightPdf(const SceneView& sc, uint lightIndex) { return float(sc.proxyCounters[lightIndex]) / float(sc.samplingProxyCount); }
PT_DEVICE float misBalance(float p0, float p1) { return sat(p0 / (p0 + p1)); }      // EvalMIS balance with n0 = n1 = 1 (Utils/Utils.hlsli:407-437)
PT_DEVICE float misForBsdf(const SceneView& sc, uint lightIndex, float bsdfPdf, float solidAnglePdf, uint fullSamples)     // ComputeLightVsBSDF_MIS_ForBSDF
{
    const float lightAvgPdf = (0.0f + globalLightPdf(sc, lightIndex)) * float(fullSamples);
    return misBalance(bsdfPdf, lightAvgPdf * solidAnglePdf);
}
// NEE-AT feedback active: the global table is the per-frame one (its total lives in device memory) and the previous vertex may also have drawn from the pixel's tile sampler
// (LightSampler.hlsli:318-333: local candidates only for screen-space-coherent vertices); misPacked = NEEBSDFMISInfo of the previous vertex
PT_DEVICE float naGlobalLightPdf(const LaunchParams& p, uint lightIndex) { return float(p.na.proxyCounters[lightIndex]) / float(*p.na.samplingProxyCount); }
template <bool NEEAT>
PT_DEVICE float misForBsdfT(const LaunchParams& p, uint pathId, uint misPacked, uint lightIndex, float bsdfPdf, float solidAnglePdf)
{
    if constexpr (!NEEAT) return misForBsdf(p.scene, lightIndex, bsdfPdf, solidAnglePdf, misPacked & 0x3F);
    else
    {
        float localPdf = 0.0f;
        if ((misPacked & (1u << 13)) && neeat::candidateLocalCount(p.na.localToGlobalSampleRatio, (misPacked >> 6) & 0x3F) > 0)
            localPdf = neeat::sampleLocalPdf(p.na, neeat::localSamplingTilePos(p.na, pathId >> 16, pathId & 0xFFFFu), lightIndex);
        const float lightAvgPdf = (localPdf + naGlobalLightPdf(p, lightIndex)) * float(misPacked & 0x3F);
        return misBalance(bsdfPdf, lightAvgPdf * solidAnglePdf);
    }
}
// Approximate MIS (RTXPT_USE_APPROXIMATE_MIS = 1, LightSampler.hlsli:271-280): the light's selection x solid-angle pdf is replaced by the constant
// RTXPT_NEEAT_MIS_APPROXIMATION_LIGHTSAMPLER_BIAS = 3 on both sides, so the BSDF side needs neither the light's index nor its record nor a sampler pdf.
// EvalMIS(Balance, fullSamples * candidates, 3, 1, bsdfPdf) on the light side, EvalMIS(Balance, 1, bsdfPdf, fullSamples * candidates, 3) on the BSDF side.
constexpr float kApproxMisLightSamplerBias = 3.0f;
PT_DEVICE float misApproxForLight(uint fullSamples, uint candidateCount, float bsdfPdf) { return misBalance(float(fullSamples * candidateCount) * kApproxMisLightSamplerBias, bsdfPdf); }
PT_DEVICE float misApproxForBsdf(uint misPacked, float bsdfPdf) { return misBalance(bsdfPdf, float((misPacked & 0x3F) * ((misPacked >> 6) & 0x3F)) * kApproxMisLightSamplerBias); }

// ---- firefly filter (PathTracerHelpers.hlsli:183-219) ----------------------------------------------------------------------------
PT_DEVICE float coneSpreadFromPdf(float pdf, float growth) { return growth * 2.0f * fastACos(fmaxf(-1.0f, 1.0f - (1.0f / pdf) / (2.0f * kPi))); }
PT_DEVICE float newFireflyK(float currentK, float bouncePdf, float lobeP)
{
    const float angle = (bouncePdf == 0) ? 0.f : coneSpreadFromPdf(bouncePdf, 1.0f);
    float q = 32.f / (32.f + angle * angle);
    q *= fastSqrt(lobeP);
    return lp(fmaxf(0.00001f, currentK * q));
}
PT_DEVICE float3 fireflyFilter(float3 signal, float threshold, float k)
{
    // lpfloat arithmetic of the reference: every operation rounds to binary16 (PathTracerHelpers.hlsli:206-212, Utils.hlsli:63-66; pinned by tests/golden/helpers_golden.npz)
    signal = lp3(signal);                                                           // the parameter is an lpfloat3
    const float thr = lp(threshold * k);
    const float maxR = lp(lp(lp(signal.x + signal.y) + signal.z) / 3.0f);
    if (maxR > thr) signal = mk3(lp(lp(signal.x / maxR) * thr), lp(lp(signal.y / maxR) * thr), lp(lp(signal.z / maxR) * thr));
    return signal;
}

// ---- surface ------------------------------------------------------------------------------------------------------------------------
struct Surface
{
    float3 posW, faceN, V, N, T, B, vertexN;
    bool frontFacing, thin;
    uint nestedPriority, materialID;
    float IoR, shadowNoLFadeout, interiorIoR;
    float3 emission;
    BsdfParams bsdf;
    uint neeTriangleLightIndex;
    uint neeAnalyticLightIndex;     // light this geometry stands in for (PTMaterialFlags_EnableAsAnalyticLightProxy), else kInvalidLight
    // path-space decomposition controls, read by realtime mode only (MaterialHeader, BridgeDonut:699-718)
    bool psdExclude, psdBlockMVs; uint psdDominantDeltaLobeP1;
    float3 prevPosW;                // BUILD pass only: instance.prevTransform x last frame's object-space position (BridgeDonut:631)
};

#ifdef PT_HOST_EMU
__host__ __device__ void emuLoadSurface(Surface& s);
#endif
PT_DEVICE float3 safeNormalize(float3 v) { return v * (1.0f / sqrtf(fmaxf(1.175494351e-38f, dot3(v, v)))); }
PT_DEVICE void computeTangentSpace(Surface& s, float4 tangentW, bool ignoreTangent)
{
    const float3 t = mk3(tangentW.x, tangentW.y, tangentW.z);
    const float NdotT = dot3(t, s.N);
    const bool valid = tangentW.w != 0.f && dot3(t, t) > 0.f && fabsf(NdotT) < 0.9999f;
    if (!ignoreTangent && valid) { s.T = norm3(t - s.N * NdotT); s.B = cross3(s.N, s.T) * tangentW.w; }
    else { s.T = perpStark(s.N); s.B = cross3(s.N, s.T); }
}

// PathTracerBridgeDonut.hlsli:104-150: RMS magnitude of the gradient of the (object-space, unit) vertex normals over the world-space triangle, 1 / position units
PT_DEVICE float triangleCurvatureGradN(const float* xf, float3 p0, float3 p1, float3 p2, float3 n0, float3 n1, float3 n2)
{
    const float eps = 1e-8f;
    const float3 e10 = xfVector(xf, p1 - p0);
    const float e10Len = len3(e10);
    if (e10Len < eps) return 0.0f;
    const float3 e1 = e10 / e10Len;
    const float3 e20 = xfVector(xf, p2 - p0);
    const float u2 = dot3(e20, e1);
    const float3 t = e20 - e1 * u2;
    const float tLen = len3(t);
    if (tLen < eps) return 0.0f;
    const float3 e2 = t / tLen;
    const float v2 = dot3(e20, e2);
    const float3 a = (n1 - n0) / fmaxf(e10Len, eps);
    const float denomV = fabsf(v2) < eps ? (v2 >= 0.0f ? eps : -eps) : v2;
    const float3 b = ((n2 - n0) - a * u2) / denomV;
    return sqrtf(dot3(a, a) + dot3(b, b));
}

// MODE: the realtime passes also need the motion-vector controls of the surface (block heuristics: every realtime pass; last frame's position: BUILD pass only); the reference-mode
// instantiation carries none of that code.  pathId = packed pixel, vertexIndex / sampleIndex seed the heuristic's MicroRng (BridgeDonut:714).
// AMIS (approximate MIS): the emissive triangle's light index is not looked up - nothing reads it (BridgeDonut:806-810).
// STF: the material textures are fetched through stochastic texture filtering (sampleMaterialTextureStf) with the vertex's sampler state (BridgeDonut:637-656).
template <int MODE, bool AMIS = false, bool STF = false>
PT_DEVICE void loadSurface(const LaunchParams& p, uint gid, float bu, float bv, float3 rayDir, float coneWidth, Surface& s, uint pathId = 0, uint vertexIndex = 1, uint sampleIndex = 0)
{
    const SceneView& sc = p.scene;
    // one contiguous 96-byte record per triangle (scene_device.cuh) instead of the reference's chain of table and vertex fetches (BridgeDonut:152-256)
    const uint4* rec = sc.triShade + size_t(gid) * kTriShadeWords;
    const uint4 r0 = __ldg(rec), r1 = __ldg(rec + 1), r2 = __ldg(rec + 2), r3 = __ldg(rec + 3), r4 = __ldg(rec + 4), r5 = __ldg(rec + 5);
    const uint4 info = make_uint4(r5.y, 0u, r5.w & kTriShadePrimMask, r5.z);          // instance, -, primitive, sub-instance
    const RtxptInstanceData& inst = sc.instances[info.x];
    const float* xf = inst.transform;
    const float b0 = 1.0f - (bu + bv);
    const float3 p0 = mk3(__uint_as_float(r0.x), __uint_as_float(r0.y), __uint_as_float(r0.z));
    const float3 p1 = mk3(__uint_as_float(r1.x), __uint_as_float(r1.y), __uint_as_float(r1.z));
    const float3 p2 = mk3(__uint_as_float(r2.x), __uint_as_float(r2.y), __uint_as_float(r2.z));
    const float3 objPos = p0 * b0 + p1 * bu + p2 * bv;
    float2 uv = mk2(0.f, 0.f), t0 = uv, t1 = uv, t2 = uv;
    if (r5.w & kTriShadeHasUV)
    {
        t0 = mk2(__uint_as_float(r3.x), __uint_as_float(r3.y)); t1 = mk2(__uint_as_float(r3.z), __uint_as_float(r3.w)); t2 = mk2(__uint_as_float(r4.x), __uint_as_float(r4.y));
        uv = mk2(t0.x * b0 + t1.x * bu + t2.x * bv, t0.y * b0 + t1.y * bu + t2.y * bv);
    }
    const float3 objFlat = safeNormalize(cross3(p1 - p0, p2 - p0));
    float3 geometryNormal = mk3(0.f);
    float curvatureWS = 0.0f;
    if (r5.w & kTriShadeHasNormal)
    {
        float3 n0 = norm3(mk3(unpackSnorm8(r0.w), unpackSnorm8(r0.w >> 8), unpackSnorm8(r0.w >> 16)));
        float3 n1 = norm3(mk3(unpackSnorm8(r1.w), unpackSnorm8(r1.w >> 8), unpackSnorm8(r1.w >> 16)));
        float3 n2 = norm3(mk3(unpackSnorm8(r2.w), unpackSnorm8(r2.w >> 8), unpackSnorm8(r2.w >> 16)));
        if (dot3(n0, objFlat) < 0) n0 = -n0;
        if (dot3(n1, objFlat) < 0) n1 = -n1;
        if (dot3(n2, objFlat) < 0) n2 = -n2;
        if (MODE != kModeReference) { const uint blockType = (sc.materials[sc.subInstances[r5.z].GlobalGeometryIndex_PTMaterialDataIndex & 0xFFFF].Flags >> 13) & 3u; if (blockType == 1u || blockType == 2u) curvatureWS = triangleCurvatureGradN(xf, p0, p1, p2, n0, n1, n2); }
        geometryNormal = safeNormalize(xfVector(xf, n0 * b0 + n1 * bu + n2 * bv));
    }
    float4 tangent = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r5.w & kTriShadeHasTangent)
    {
        const uint q0 = r4.z, q1 = r4.w, q2 = r5.x;
        const float3 a = mk3(unpackSnorm8(q0), unpackSnorm8(q0 >> 8), unpackSnorm8(q0 >> 16));
        const float3 b = mk3(unpackSnorm8(q1), unpackSnorm8(q1 >> 8), unpackSnorm8(q1 >> 16));
        const float3 c = mk3(unpackSnorm8(q2), unpackSnorm8(q2 >> 8), unpackSnorm8(q2 >> 16));
        const float3 txyz = safeNormalize(xfVector(xf, a * b0 + b * bu + c * bv));
        tangent = make_float4(txyz.x, txyz.y, txyz.z, unpackSnorm8(q0 >> 24));
    }
    const float3 flatNormal = safeNormalize(xfVector(xf, objFlat));
    const bool frontFacing = dot3(-rayDir, flatNormal) >= 0.0f;

    s.posW = xfPoint(xf, objPos);
    if (MODE == kModeBuildStablePlanes)
    {   // GeomAttr_PrevPosition (BridgeDonut:187-199, :631)
        float3 prevObj = objPos;
        const uint base = sc.prevPosBase ? __ldg(sc.prevPosBase + r5.z) : 0xFFFFFFFFu;
        if (base != 0xFFFFFFFFu)
        {
            const float* q = sc.triPrevPos + (size_t(base) + (r5.w & kTriShadePrimMask)) * 9;
            prevObj = mk3(__ldg(q), __ldg(q + 1), __ldg(q + 2)) * b0 + mk3(__ldg(q + 3), __ldg(q + 4), __ldg(q + 5)) * bu + mk3(__ldg(q + 6), __ldg(q + 7), __ldg(q + 8)) * bv;
        }
        s.prevPosW = xfPoint(inst.prevTransform, prevObj);
    }
    // ray-cone LOD: computeRayConeTriangleLODValue + RayCone::computeLOD(moreDetailOnSlopes) + texLODBias
    float lodNoDims;
    {
        const float Ta = fabsf((t1.x - t0.x) * (t2.y - t0.y) - (t2.x - t0.x) * (t1.y - t0.y));
        const float Pa = len3(cross3(xfVector(xf, p1 - p0), xfVector(xf, p2 - p0)));
        const float triLOD = 0.5f * safeLog2(Ta / Pa);
        const float normalTerm = sqrtf(fabsf(dot3(rayDir, flatNormal)));
        lodNoDims = triLOD + safeLog2(fabsf(coneWidth) / normalTerm) + p.c.texLODBias;
    }
    s.V = -rayDir;
    s.N = geometryNormal;
    const uint subIndex = info.w;
    const uint materialIndex = sc.subInstances[subIndex].GlobalGeometryIndex_PTMaterialDataIndex & 0xFFFF;
    const RtxptMaterialData& m = sc.materials[materialIndex];
    const uint mflags = m.Flags;

    // sampleGeometryMaterialRTXPT + EvaluateSceneMaterialRTXPT
    float4 texBase = make_float4(1, 1, 1, 1), texMR = texBase, texEmissive = texBase, texNormal = make_float4(0.5f, 0.5f, 1.0f, 0.0f);
    float texTrans = 1.0f;
    if constexpr (STF)
    {   // the bridge's five fetches in its order and under its conditions (BridgeDonut:402-423)
        StfState stf;
        stf.u = stfVertexRandom(pathId, vertexIndex, sampleIndex);
        stf.filterType = p.stf.filterType; stf.sigma = p.stf.sigma; stf.reseedOnSample = false;
        if (mflags & RTXPT_MATFLAG_UseBaseOrDiffuseTexture) texBase = sampleMaterialTextureStf(p, m.BaseOrDiffuseTextureIndex, lodNoDims, uv, stf);
        if (mflags & RTXPT_MATFLAG_UseEmissiveTexture) texEmissive = sampleMaterialTextureStf(p, m.EmissiveTextureIndex, lodNoDims, uv, stf);
        if (mflags & RTXPT_MATFLAG_UseNormalTexture) texNormal = sampleMaterialTextureStf(p, m.NormalTextureIndex, lodNoDims, uv, stf);
        if (mflags & RTXPT_MATFLAG_UseMetalRoughOrSpecularTexture) texMR = sampleMaterialTextureStf(p, m.MetalRoughOrSpecularTextureIndex, lodNoDims, uv, stf);
        if (mflags & RTXPT_MATFLAG_UseTransmissionTexture) texTrans = sampleMaterialTextureStf(p, m.TransmissionTextureIndex, lodNoDims, uv, stf).x;
    }
    else
    {
        if (mflags & RTXPT_MATFLAG_UseBaseOrDiffuseTexture) texBase = sampleMaterialTexture(sc, m.BaseOrDiffuseTextureIndex, lodNoDims, uv);
        if (mflags & RTXPT_MATFLAG_UseEmissiveTexture) texEmissive = sampleMaterialTexture(sc, m.EmissiveTextureIndex, lodNoDims, uv);
        if (mflags & RTXPT_MATFLAG_UseNormalTexture) texNormal = sampleMaterialTexture(sc, m.NormalTextureIndex, lodNoDims, uv);
        if (mflags & RTXPT_MATFLAG_UseMetalRoughOrSpecularTexture) texMR = sampleMaterialTexture(sc, m.MetalRoughOrSpecularTextureIndex, lodNoDims, uv);
        if (mflags & RTXPT_MATFLAG_UseTransmissionTexture) texTrans = sampleMaterialTexture(sc, m.TransmissionTextureIndex, lodNoDims, uv).x;
    }

    const float3 matGeometryNormal = norm3(geometryNormal);
    float3 shadingNormal = matGeometryNormal;
    float3 baseColor; float roughness, metalness;
    const float3 baseFactor = mk3(m.BaseOrDiffuseColor[0], m.BaseOrDiffuseColor[1], m.BaseOrDiffuseColor[2]);
    if (mflags & RTXPT_MATFLAG_UseSpecularGlossModel)
    {   // ConvertSpecularGlossToMetalRough (External/Donut/include/donut/shaders/scene_material.hlsli:88-117)
        const float3 diffuseColor = baseFactor * mk3(texBase.x, texBase.y, texBase.z);
        const float3 specularColor = mk3(m.SpecularColor[0], m.SpecularColor[1], m.SpecularColor[2]) * mk3(texMR.x, texMR.y, texMR.z);
        roughness = lp(1.0f - texMR.w * (1.0f - m.Roughness));
        const float oneMinusSpec = 1.0f - maxComp(specularColor);
        const float dB = sqrtf(0.299f * diffuseColor.x * diffuseColor.x + 0.587f * diffuseColor.y * diffuseColor.y + 0.114f * diffuseColor.z * diffuseColor.z);
        const float sB = sqrtf(0.299f * specularColor.x * specularColor.x + 0.587f * specularColor.y * specularColor.y + 0.114f * specularColor.z * specularColor.z);
        float metal = 0.f;
        if (!(sB < 0.04f))
        {
            const float a = 0.04f, b = dB * oneMinusSpec / (1 - 0.04f) + sB - 2 * 0.04f, c = 0.04f - sB;
            metal = clampf((-b + sqrtf(fmaxf(b * b - 4 * a * c, 0.f))) / (2 * a), 0.f, 1.f);
        }
        const float3 fromDiffuse = diffuseColor * (oneMinusSpec / (1 - 0.04f) / fmaxf(1 - metal, 1e-6f));
        const float3 fromSpecular = specularColor - mk3(0.04f * (1 - metal) / fmaxf(metal, 1e-6f));
        baseColor = lp3(sat3(lerp3(fromDiffuse, fromSpecular, metal * metal)));
        metalness = lp(metal);
    }
    else
    {
        baseColor = lp3(baseFactor * mk3(texBase.x, texBase.y, texBase.z));
        roughness = lp(m.Roughness * texMR.y);
        metalness = lp(m.Metalness * ((mflags & RTXPT_MATFLAG_MetalnessInRedChannel) ? texMR.x : texMR.z));
    }
    float transmission = lp(m.TransmissionFactor), diffuseTransmission = lp(m.DiffuseTransmissionFactor);
    if (mflags & RTXPT_MATFLAG_UseTransmissionTexture) { transmission = lp(transmission * lp(texTrans)); diffuseTransmission = lp(diffuseTransmission * lp(texTrans)); }
    float3 emissiveColor = lp3(mk3(m.EmissiveColor[0], m.EmissiveColor[1], m.EmissiveColor[2]));
    if (mflags & RTXPT_MATFLAG_UseEmissiveTexture) emissiveColor = lp3(emissiveColor * lp3(mk3(texEmissive.x, texEmissive.y, texEmissive.z)));
    const float matIoR = lp(m.IoR);
    if (mflags & RTXPT_MATFLAG_UseNormalTexture)
    {   // ApplyNormalMapRTXPT (BridgeDonut:280-309)
        const float sqT = tangent.x * tangent.x + tangent.y * tangent.y + tangent.z * tangent.z;
        if (sqT != 0 && tangent.w != 0)
        {
            const float nx = (texNormal.x * 2.0f - 1.0f) * m.NormalTextureScale, ny = (texNormal.y * 2.0f - 1.0f) * m.NormalTextureScale;
            const float nz = (texNormal.z <= 0) ? sqrtf(sat(1.0f - nx * nx - ny * ny)) : fabsf(texNormal.z * 2.0f - 1.0f);
            const float sqLen = nx * nx + ny * ny + nz * nz;
            if (sqLen != 0)
            {
                const float len = sqrtf(sqLen);
                const float3 t = mk3(tangent.x, tangent.y, tangent.z) * (1.0f / sqrtf(sqT));
                const float3 bitangent = cross3(matGeometryNormal, t) * tangent.w;
                shadingNormal = norm3(t * (nx / len) + bitangent * (ny / len) + matGeometryNormal * (nz / len));
            }
        }
    }
    const bool ignoreTangent = (mflags & RTXPT_MATFLAG_IgnoreMeshTangentSpace) != 0;
    // (the reference also builds a tangent frame around the geometry normal here; adjustShadingNormal below rebuilds it, so it is skipped)
    s.faceN = frontFacing ? flatNormal : -flatNormal;
    s.vertexN = frontFacing ? geometryNormal : -geometryNormal;
    s.frontFacing = frontFacing;
    s.N = frontFacing ? shadingNormal : -shadingNormal;
    s.materialID = materialIndex;
    s.nestedPriority = min(15u, 1u + (mflags >> RTXPT_MATFLAG_NestedPriorityShift));
    s.thin = (mflags & RTXPT_MATFLAG_ThinSurface) != 0;
    s.psdExclude = (mflags & RTXPT_MATFLAG_PSDExclude) != 0;
    s.psdDominantDeltaLobeP1 = (mflags & 0x0F000000u) >> 24;
    {   // stopping motion vectors behind this surface (BridgeDonut:702-718): 0 Off, 1 AutoLow, 2 AutoHigh (triangle curvature seen through the ray cone), 3 Full
        const uint blockType = (mflags >> 13) & 3u;
        s.psdBlockMVs = blockType == 3u;
        if (MODE != kModeReference && (blockType == 1u || blockType == 2u))
        {
            const float projectionTerm = fabsf(dot3(rayDir, -s.N));
            const float pixelCurvature = (curvatureWS * coneWidth) / fmaxf(projectionTerm, 1e-6f);
            neeat::MicroRng rng = neeat::MicroRng::make(pathId >> 16, pathId & 0xFFFFu, vertexIndex, sampleIndex);
            s.psdBlockMVs = pixelCurvature > ((rng.nextFloat() * 0.9f + 0.3f) * (blockType == 1u ? 0.03f : 0.0005f));
        }
    }
    {   // adjustShadingNormal(recomputeTangentSpace = true)
        const float signN = dot3(s.N, s.faceN) >= 0.f ? 1.f : -1.f;
        const float3 Ns = signN * s.N;
        const float cosTheta = dot3(s.V, Ns);
        if (cosTheta <= 0.1f) s.N = signN * norm3(lerp3(s.faceN, Ns, sat(cosTheta * (1.f / 0.1f))));
        computeTangentSpace(s, tangent, ignoreTangent);
    }
    s.shadowNoLFadeout = lp(m.ShadowNoLFadeout);
    s.bsdf.specularTransmission = lp(transmission * (1 - metalness));
    s.bsdf.diffuseTransmission = lp(diffuseTransmission * (1 - metalness));
    s.bsdf.transmission = baseColor;
    const float f = (matIoR - 1.f) / (matIoR + 1.f);
    const float F0 = f * f;
    s.bsdf.diffuse = lp3(lerp3(baseColor, mk3(0.f), metalness));
    s.bsdf.specular = lp3(lerp3(lp3(mk3(F0)), baseColor, metalness));
    s.bsdf.roughness = roughness;
    s.bsdf.metallic = metalness;
    s.IoR = 1.f;
    s.bsdf.eta = lp(s.IoR / matIoR);
    if (!s.thin && !frontFacing) s.bsdf.eta = lp(matIoR / s.IoR);
    s.neeTriangleLightIndex = kInvalidLight;
    s.neeAnalyticLightIndex = (mflags & RTXPT_MATFLAG_EnableAsAnalyticLightProxy) ? sc.subInstances[subIndex].AnalyticProxyLightIndex : kInvalidLight;      // BridgeDonut:828-829
    s.emission = mk3(0.f);
    if (frontFacing && anyPositive(emissiveColor))
    {
        s.emission = emissiveColor;
        if constexpr (!AMIS)
        {
            const uint baseIndex = sc.subInstances[subIndex].EmissiveLightMappingOffset;
            if (baseIndex != 0xFFFFFFFFu) s.neeTriangleLightIndex = baseIndex + info.z;
        }
    }
    s.interiorIoR = matIoR;
}

// ---- interior list (InteriorList.hlsli, 2 slots) --------------------------------------------------------------------------------------
constexpr uint kInteriorMaterialMask = (1u << 28) - 1u;
PT_DEVICE void interiorHandleIntersection(PathRegs& path, uint materialID, uint nestedPriority, bool entering)
{
    if (nestedPriority == 0) nestedPriority = 15;
    const uint slot = (nestedPriority << 28) | (materialID & kInteriorMaterialMask);
    uint& s0 = path.interior0; uint& s1 = path.interior1;
    if (entering && s0 == 0) s0 = slot;
    else if (!entering && s0 != 0 && (s0 & kInteriorMaterialMask) == materialID) s0 = 0;
    else if (entering && s1 == 0) s1 = slot;
    else if (!entering && s1 != 0 && (s1 & kInteriorMaterialMask) == materialID) s1 = 0;
    if (s0 < s1) { const uint t = s0; s0 = s1; s1 = t; }
}

// ---- miss ---------------------------------------------------------------------------------------------------------------------------------
PT_DEVICE void updatePathTravelled(PathRegs& path, float rayT)      // PathTracer.hlsli:382-404
{
    path.flagsAndVertexIndex += 1;
    const float angle = path.coneSpread(), width = path.coneWidth();
    path.setCone(angle * rayT + width, angle);
    path.sceneLength = fminf(path.sceneLength + rayT, kMaxRayTravel);
}

} // namespace pt
#include "realtime.cuh"
namespace pt {

// AccumulatePathRadiance (PathTracer.hlsli:139-162)
template <int MODE>
PT_DEVICE void accumulatePathRadiance(const LaunchParams& p, PathRegs& path, float3 radiance)
{
    if constexpr (MODE == kModeReference) path.addRadiance(radiance);
    else if constexpr (MODE == kModeBuildStablePlanes) accumulateStableRadiance(p, path.id, radiance);
    else if (!path.hasFlag(kPFStablePlaneOnBranch))         // FILL: what lies on the stable branches was captured by the BUILD pass
    {
        const float specAvg = path.hasFlag(kPFStablePlaneBaseScatterDiff) ? 0.0f : average(radiance);
        const float a = p.rt.attenuation; const float4 l = path.L();
        path.setL(make_float4(l.x + radiance.x * a, l.y + radiance.y * a, l.z + radiance.z * a, l.w + specAvg * a));
    }
}

// AMIS: approximate light-vs-BSDF MIS (RTXPT_USE_APPROXIMATE_MIS = 1) at the environment miss, the emissive triangle, the analytic proxy and the light sample
template <bool EXPORT_GUIDES, int MODE = kModeReference, bool NEEAT = false, bool AMIS = false>
PT_DEVICE void shadeMiss(const LaunchParams& p, PathRegs& path)
{
    const float3 segmentOrigin = path.origin;
    updatePathTravelled(path, kMaxRayTravel);
    if constexpr (MODE == kModeFillStablePlanes) if (path.hasFlag(kPFExportSpecHitTQueued)) { exportSpecHitTStop(p, path); path.setFlag(kPFExportSpecHitTQueued, false); }
    float3 emission = mk3(0.f);
    if (p.scene.envEnabled)
    {
        const uint mis = (MODE == kModeBuildStablePlanes) ? 0u : path.misInfo();      // no NEE, no MIS while the planes are built (PathState.hlsli:157-159)
        const float mip = (path.counter(kCtrDiffuseBounces) > 1) ? p.c.EnvironmentMapDiffuseSampleMIPLevel : 0.0f;
        const float3 localDir = rowVecTimes3x3(path.dir, p.c.envMap.InvTransform);
        const float3 Le = envEvalLocal(p, localDir, mip);
        float misWeight = 1.0f;
        const float bsdfPdf = (MODE == kModeBuildStablePlanes) ? 0.0f : path.bsdfScatterPdf();
        if constexpr (AMIS) { if ((mis & (1u << 15)) && bsdfPdf != 0) misWeight = misApproxForBsdf(mis, bsdfPdf); }         // PathTracer.hlsli:461-462: no quad-tree lookup
        else if ((mis & (1u << 15)) && bsdfPdf != 0)
        {
            const float2 uv = dirToOctEqualArea(localDir);
            const uint cx = min(uint(uv.x * float(kEnvLookupDim)), kEnvLookupDim - 1), cy = min(uint(uv.y * float(kEnvLookupDim)), kEnvLookupDim - 1);
            const uint li = p.scene.envLookupMap[cy * kEnvLookupDim + cx];
            const uint nodeDim = p.scene.lights[li].direction2 >> 16;
            misWeight = misForBsdfT<NEEAT>(p, path.id, mis, li, bsdfPdf, float(nodeDim * nodeDim) / (4.0f * kPi));
        }
        emission = lp3(misWeight * Le);
    }
    const float ffThreshold = lp(p.c.fireflyFilterThreshold);
    if (MODE != kModeBuildStablePlanes && ffThreshold != 0) emission = fireflyFilter(emission, ffThreshold, path.fireflyK());
    if constexpr (MODE == kModeBuildStablePlanes) stablePlanesHandleMiss(p, path, emission, segmentOrigin, path.dir);
    if constexpr (MODE == kModeReference) if (EXPORT_GUIDES && path.sampleIndex + 1 == p.firstSampleIndex + p.subSampleCount)
        exportGuide(p, path.id, path.origin + path.dir * kMaxRayTravel, 0u);                 // ExportNonSurface (PathTracer.hlsli:487)
    if (anyPositive(emission)) accumulatePathRadiance<MODE>(p, path, path.thp() * emission);
    path.setFlag(kPFHit, false);
    path.setFlag(kPFActive, false);
}

// ---- hit -----------------------------------------------------------------------------------------------------------------------------------
struct HitOutputs { bool continuePath; bool emitShadow; ShadowRecord shadow; uint4 naRecord; };     // naRecord: NEE-AT feedback of the shadow record (kernels with NEEAT = true)

// FILL pass: which specular average AccumulatePathRadiance adds with the NEE radiance (PathTracer.hlsli:731-743), as the sign bits of the first word of the packed
// (radiance, specAvg) - whose halves are non-negative: 00 none (the base scatter was diffuse), 01 the NEE result's own, 10 the average of the radiance.  ORed into `word`.
PT_DEVICE void addFillSpecAvgChoice(uint& word, uint preFlags, uint preCounters)
{
    if (!(preFlags & (kPFStablePlaneBaseScatterDiff << kVertexIndexBits)))
    {
        const uint bouncesFromStablePlane = ((preCounters >> (kCtrBouncesFromStablePlane << 3)) & 0xffu) + 1u;
        const bool special = (bouncesFromStablePlane == 1) || ((preFlags & (kPFDeltaOnlyPath << kVertexIndexBits)) && bouncesFromStablePlane <= 3);
        word |= special ? 0x00008000u : 0x80000000u;
    }
}

// surfaceDebugViz (PathTracerBridgeDonut.hlsli:457-510, called at the end of Bridge::loadSurface): the first-hit debug view from the surface just loaded
PT_DEVICE void storeFirstHitDebugView(const LaunchParams& p, uint id, float bu, float bv, const Surface& s)
{
    FirstHitDebugInputs d;
    d.barycentrics = mk2(bu, bv);
    d.faceN = s.faceN; d.vertexN = s.vertexN; d.N = s.N; d.T = s.T; d.B = s.B;
    d.frontFacing = s.frontFacing; d.thin = s.thin;
    d.diffuse = s.bsdf.diffuse; d.specular = s.bsdf.specular; d.roughness = s.bsdf.roughness; d.metallic = s.bsdf.metallic;
    d.materialID = s.materialID;
    p.dbg.viz[pixelOffset(p, id)] = packDebugPixel(firstHitDebugColor(p.dbg.view, d));
}

// MULTI: NEEFullSamples > 1 - the light samples' shadow records and the vertex's NEE block go straight to the launch's arrays (out.emitShadow stays false).  Without
// NEE-AT feedback no draw depends on visibility, so the samples are drawn one after the other from the vertex's one uniform stream as HandleNEE draws them.
// DEBUG_VIEW: a first-hit debug view is set (LaunchParams::dbg); vertex 1 draws it - in reference mode only in the call's last sub-sample, whose value RTXPT's last dispatch leaves
template <bool EXPORT_GUIDES, bool ANALYTIC_LIGHTS, int MODE = kModeReference, bool NEEAT = false, bool MULTI = false, bool AMIS = false, bool STF = false, bool DEBUG_VIEW = false>
PT_DEVICE void shadeHit(const LaunchParams& p, PathRegs& path, uint slot, float4 hit, HitOutputs& out)
{
    out.continuePath = false; out.emitShadow = false;
    constexpr bool kBuild = MODE == kModeBuildStablePlanes, kFill = MODE == kModeFillStablePlanes;
    if constexpr (NEEAT)
    {   // The previous vertex's light sample turned out visible: its feedback insertion drew one more number of the vertex's uniform sequence before Russian roulette did
        // (PathTracerNEE.hlsli:276-283, PathTracer.hlsli:182-208).  Visibility is only known after the shadow kernel, so that vertex stored both roulette outcomes: the path
        // state holds the "not visible" one, the shadow kernel published the other one here.
        const uint fix = p.naRrFix[slot];
        if (fix & 0x80000000u)
        {
            path.setFlag(kPFTerminateAtNextBounce, (fix & 0x40000000u) != 0);
            path.setMisInfo_RuRu(path.misInfo(), f16tof32(fix & 0xFFFFu));
            p.naRrFix[slot] = 0;
        }
    }
    const uint sampleIndex = (MODE == kModeReference) ? path.sampleIndex : p.firstSampleIndex;      // realtime passes: one sample index per launch, the word holds stableBranchID
    const float3 rayOrigin = path.origin, rayDir = path.dir;
    const float rayT = hit.x;
    updatePathTravelled(path, rayT);
    Surface s;
#ifdef PT_HOST_EMU
    emuLoadSurface(s);
#else
    loadSurface<MODE, AMIS, STF>(p, __float_as_uint(hit.w), hit.y, hit.z, rayDir, path.coneWidth(), s, path.id, path.vertexIndex(), sampleIndex);
#endif
    if constexpr (DEBUG_VIEW)
        if (path.vertexIndex() == 1 && (MODE != kModeReference || path.sampleIndex + 1 == p.firstSampleIndex + p.subSampleCount)) storeFirstHitDebugView(p, path.id, hit.y, hit.z, s);
    const uint ndq = p.c.nestedDielectricsQuality;
    if (ndq > 0 && path.interior0 != 0)
    {   // homogeneous absorption through the medium we are in (PathTracer.hlsli:538-547, BridgeDonut:871-887)
        const uint materialID = path.interior0 & kInteriorMaterialMask;
        float3 sigmaA = mk3(0.f);
        if (materialID < p.scene.materialCount)
        {
            const RtxptMaterialData& vm = p.scene.materials[materialID];
            const float dist = fmaxf(1e-30f, vm.VolumeAttenuationDistance);
            sigmaA = mk3(-logf(clampf(vm.VolumeAttenuationColor[0], 1e-7f, 1.f)) / dist, -logf(clampf(vm.VolumeAttenuationColor[1], 1e-7f, 1.f)) / dist, -logf(clampf(vm.VolumeAttenuationColor[2], 1e-7f, 1.f)) / dist);
        }
        path.setThp(path.thp() * mk3(expf(-rayT * sigmaA.x), expf(-rayT * sigmaA.y), expf(-rayT * sigmaA.z)));
    }
    if (ndq > 0 && !s.thin)
    {   // HandleNestedDielectrics, quality 1 (4 rejected hits, no termination)
        const uint topPriority = path.interior0 >> 28;
        const bool trueIntersection = s.nestedPriority == 0 || s.nestedPriority >= topPriority;
        if (path.counter(kCtrRejectedHits) < 4 && !trueIntersection)
        {
            path.incrementCounter(kCtrRejectedHits);
            interiorHandleIntersection(path, s.materialID, s.nestedPriority, s.frontFacing);
            path.origin = offsetRayOrigin(s.posW, -s.faceN);
            path.flagsAndVertexIndex -= 1;
            out.continuePath = true;        // false hit: continue along the same direction from the far side
            return;
        }
        uint outsideMaterial = (path.interior0 != 0) ? (path.interior0 & kInteriorMaterialMask) : 0xFFFFFFFFu;
        if (!s.frontFacing && outsideMaterial == s.materialID) outsideMaterial = (path.interior1 != 0) ? (path.interior1 & kInteriorMaterialMask) : 0xFFFFFFFFu;
        float outsideIoR = 1.f;
        if (outsideMaterial != 0xFFFFFFFFu) outsideIoR = (outsideMaterial >= p.scene.materialCount) ? 1.0f : lp(p.scene.materials[outsideMaterial].IoR);
        s.IoR = outsideIoR;
        s.bsdf.eta = lp(s.frontFacing ? (s.IoR / s.interiorIoR) : (s.interiorIoR / s.IoR));
    }

    // emission + BSDF-side MIS (PathTracer.hlsli:592-674)
    const uint misPacked = kBuild ? 0u : path.misInfo();
    const float pathBsdfPdf = kBuild ? 0.0f : path.bsdfScatterPdf();
    float3 surfaceEmission = mk3(0.f);
    if (anyPositive(s.emission))
    {
        float misWeight = 1.0f;
        const float bsdfPdf = pathBsdfPdf;
        // approximate MIS weights every emitter on the BSDF side, one without a light record too (ExcludeFromNEE, light-list overflow): PathTracer.hlsli:619-620 tests no index
        if constexpr (AMIS) { if ((misPacked & (1u << 15)) && bsdfPdf != 0) misWeight = misApproxForBsdf(misPacked, bsdfPdf); }
        else if ((misPacked & (1u << 15)) && bsdfPdf != 0 && s.neeTriangleLightIndex != kInvalidLight)
        {
            TriLight tl; tl.decode(p.scene.lights[s.neeTriangleLightIndex]);
            misWeight = misForBsdfT<NEEAT>(p, path.id, misPacked, s.neeTriangleLightIndex, bsdfPdf, tl.solidAnglePdfForMIS(rayOrigin, s.posW));
        }
        surfaceEmission = lp3(s.emission * misWeight);
    }
    if (ANALYTIC_LIGHTS && s.neeAnalyticLightIndex != kInvalidLight)
    {   // LightSampler::ComputeAnalyticLightProxyContributionWithMIS (LightSampler.hlsli:363-394): a BSDF ray that reached the proxy geometry
        // of a sphere light sees the analytic sphere (SphereLight::Eval + IntersectRaySphere, Utils/Geometry.hlsli:85-118)
        const LightInfo li = p.scene.lights[s.neeAnalyticLightIndex];
        if (lightType(li) == kLightTypeSphere)
        {
            const float3 center = mk3(li.cx, li.cy, li.cz); const float radius = f16tof32(li.scalars);
            const float3 lv = center - rayOrigin, oc = rayOrigin - center;
            const float bq = 2.0f * dot3(oc, rayDir), cq = dot3(oc, oc) - radius * radius, disc = bq * bq - 4.0f * cq;
            if (!(dot3(lv, lv) < radius * radius) && disc >= 0.0f)
            {
                const float sq = sqrtf(disc), t1 = (-bq - sq) / 2.0f, t2 = (-bq + sq) / 2.0f;
                if (t1 >= 0.0f || t2 >= 0.0f)
                {
                    const float3 radiance = unpackLightRadiance(li) * lightShaping(li, p.scene, s.neeAnalyticLightIndex, rayOrigin, center);
                    float mis = 1.0f;
                    const float bsdfPdf = (misPacked & (1u << 15)) ? pathBsdfPdf : 0.0f;
                    if (AMIS && bsdfPdf != 0) mis = misApproxForBsdf(misPacked, bsdfPdf);
                    else if (bsdfPdf != 0)
                    {
                        const float cosThetaMax = sqrtf(fmaxf(0.0f, 1.0f - (radius * radius) / dot3(lv, lv)));
                        mis = misForBsdfT<NEEAT>(p, path.id, misPacked, s.neeAnalyticLightIndex, bsdfPdf, 1.0f / (2.0f * kPi * (1.0f - cosThetaMax)));
                    }
                    surfaceEmission = surfaceEmission + lp3(radiance * mis);
                }
            }
        }
    }
    if (anyPositive(surfaceEmission))
    {
        const float ffThreshold = lp(p.c.fireflyFilterThreshold);
        if (!kBuild && ffThreshold != 0) surfaceEmission = fireflyFilter(surfaceEmission, ffThreshold, path.fireflyK());
        if (anyPositive(surfaceEmission)) accumulatePathRadiance<MODE>(p, path, path.thp() * surfaceEmission);
    }
    if constexpr (MODE == kModeReference) if (EXPORT_GUIDES && path.sampleIndex + 1 == p.firstSampleIndex + p.subSampleCount)
    {   // ExportSurface (PathTracer.hlsli:684): virtual position along the pixel's camera ray at the path's scene length, throughput before this vertex
        float3 co, cd; computeCameraRay(p.c, path.id, path.sampleIndex, co, cd);
        exportGuide(p, path.id, co + cd * path.sceneLength, packR11G11B10(mk3(sat(path.thp().x), sat(path.thp().y), sat(path.thp().z))));
    }
    const bool pathStopping = path.hasFlag(kPFTerminateAtNextBounce);
    if constexpr (kBuild)
    {   // the BUILD pass consumes the emission and either re-aims the path along a delta lobe or stores the plane and stops (PathTracer.hlsli:679-699)
        BsdfSetup deltaBsdf; deltaBsdf.init(s.T, s.B, s.N, s.V, s.thin, s.bsdf);
        stablePlanesHandleHit(p, path, rayOrigin, rayDir, rayT, s, deltaBsdf, pathStopping);
        if (pathStopping) { path.setFlag(kPFActive, false); return; }
        path.setThp(path.thp() * 1.0f);
        out.continuePath = path.hasFlag(kPFActive);
        return;
    }
    if (pathStopping) { path.setFlag(kPFActive, false); return; }

    path.setThp(path.thp() * path.ruRuCorrection());

    const uint baseHash = vertexBaseHash(path.id, path.vertexIndex());
    UniformSeq uniformSG = UniformSeq::make(baseHash, sampleIndex, 0u);
    // state of the path before scattering, needed by NEE
    const float3 preThp = path.thp();
    const float preFireflyK = path.fireflyK();
    const float preConeWidth = path.coneWidth(), preSceneLength = path.sceneLength;
    const uint preFlags = path.flagsAndVertexIndex, preCounters = path.packedCounters;          // preScatterPath's flags (realtime mode's classification of NEE radiance)

    BsdfSetup bsdf; bsdf.init(s.T, s.B, s.N, s.V, s.thin, s.bsdf);

    // GenerateScatterRay (PathTracer.hlsli:217-380)
    bool scatterValid;
    {
        float u0, u1, u2;
        if (p.c.enableLDSamplerForBSDF && path.counter(kCtrDiffuseBounces) < 1)
        {
            u0 = hashToFloat(ldSampleBits(baseHash, sampleIndex, 1u, 0));
            u1 = hashToFloat(ldSampleBits(baseHash, sampleIndex, 1u, 1));
            u2 = hashToFloat(ldSampleBits(baseHash, sampleIndex, 1u, 2));
        }
        else
        {
            UniformSeq sg = UniformSeq::make(baseHash, sampleIndex, 1u);
            u0 = sg.next(); u1 = sg.next(); u2 = sg.next();
        }
        BsdfSample bs;
        scatterValid = bsdf.sample(u0, u1, u2, bs);
        if (scatterValid)
        {
            path.dir = bs.wo;
            const bool onDominantDenoisingLayer = kFill && path.hasFlag(kPFStablePlaneOnPlane) && path.hasFlag(kPFStablePlaneOnDominantBranch);
            path.setThp(path.thp() * bs.weight);
            path.flagsAndVertexIndex &= ~((kPFTransmission | kPFSpecular | kPFDelta) << kVertexIndexBits);
            path.origin = offsetRayOrigin(s.posW, (bs.lobe & kLobeReflection) ? s.faceN : -s.faceN);
            const bool isDiffuse = (bs.lobe & (kLobeDiffuseReflection | kLobeDiffuseTransmission)) || s.bsdf.roughness > 0.25f;
            if (isDiffuse) { if (!((bs.lobe & kLobeDiffuseTransmission) && ((path.vertexIndex() % 2) == 1))) path.incrementCounter(kCtrDiffuseBounces); }
            else path.setFlag(kPFSpecular, true);
            if (bs.lobe & kLobeTransmission)
            {
                path.setFlag(kPFTransmission, true);
                if (ndq > 0 && !s.thin)
                {
                    interiorHandleIntersection(path, s.materialID, s.nestedPriority, s.frontFacing);
                    path.setFlag(kPFInsideDielectric, path.interior0 != 0);
                }
            }
            if (bs.lobe & kLobeDelta) path.setFlag(kPFDelta, true);
            else
            {
                path.setFlag(kPFDeltaOnlyPath, false);
                path.setCone(path.coneWidth(), fminf(path.coneSpread() + coneSpreadFromPdf(bs.pdf, 0.3f), 2.0f * kPi));
            }
            if constexpr (kFill)
            {   // specular hit distance of the dominant plane for the denoiser (PathTracer.hlsli:295-324)
                const bool isDiffuseForSpecHitT = (bs.lobe & (kLobeDiffuseReflection | kLobeDiffuseTransmission)) || s.bsdf.roughness > 0.35f;
                if (onDominantDenoisingLayer && !isDiffuseForSpecHitT)
                {
                    if (!s.psdBlockMVs) { path.setFlag(kPFExportSpecHitTQueued, true); p.rt.specularHitT[pixelOffset(p, path.id)] = -path.sceneLength; }     // ExportSpecHitTStart
                }
                else if (path.hasFlag(kPFExportSpecHitTQueued))
                {
                    if ((bsdfLobes(s.bsdf) & kLobeNonDelta) != 0 || path.counter(kCtrBouncesFromStablePlane) > 4) { exportSpecHitTStop(p, path); path.setFlag(kPFExportSpecHitTQueued, false); }
                }
            }
            const float k = (p.c.fireflyFilterThreshold != 0) ? newFireflyK(path.fireflyK(), bs.pdf, bs.lobeP) : 0.0f;
            path.setFireflyK_BsdfPdf(k, bs.pdf);
            if constexpr (kFill) stablePlanesOnScatter(p, path, bs.lobe);
            path.setFlag(kPFEnableThreadReorder, true);
        }
    }

    // HandleNEE (PathTracerNEE.hlsli:303-346): per light sample, candidates by weighted reservoir sampling and one shadow ray
    uint neeMis = 0;
    const uint fullSamples = min(kNeeMaxFullSamples, p.c.NEEFullSamples);      // kernels without MULTI run with NEEFullSamples <= 1 (the reference default): one shadow record per vertex
    uint naFeedback = 0xFFFFFFFFu; float naFeedbackWeight = 0.0f;          // NEEAT: the picked light (| ssc << 31) and how much the pixel wanted it
    if (p.c.NEEEnabled && (bsdfLobes(s.bsdf) & kLobeNonDelta) != 0 && (NEEAT ? *p.na.samplingProxyCount : p.scene.samplingProxyCount) != 0 && fullSamples > 0)
    {
        const uint candidateCount = p.c.NEECandidateSamples;
        const bool isSSC = (preConeWidth / preSceneLength) < (NEEAT ? p.na.screenSpaceVsWorldSpaceThreshold : 0.3f);
        neeMis = (1u << 15) | ((isSSC ? 1u : 0u) << 13) | ((candidateCount & 0x3F) << 6) | (fullSamples & 0x3F);
        const uint M = NEEAT ? *p.na.samplingProxyCount : p.scene.samplingProxyCount;
        const uint* __restrict__ proxyIndices = NEEAT ? p.na.proxyIndices : p.scene.proxyIndices;
        const uint* __restrict__ proxyCounters = NEEAT ? p.na.proxyCounters : p.scene.proxyCounters;
        // GetCandidateSampleCounts: the first globalCount candidates come from the global table, the rest from the pixel's tile sampler (screen-space-coherent vertices, once
        // a frame of feedback has built the samplers)
        const uint localCount = (NEEAT && isSSC) ? neeat::candidateLocalCount(p.na.localToGlobalSampleRatio, candidateCount) : 0u, globalCount = candidateCount - localCount;
        const uint tileAddress = NEEAT ? neeat::localSamplingTilePos(p.na, path.id >> 16, path.id & 0xFFFFu) : 0u;
        uint* ctr = nullptr; uint block = 0;
        if constexpr (MULTI)
        {   // the vertex's NEE block: header now, one fp32 result per valid sample below
            ctr = p.wf.counters + p.iteration * kCountersPerIter;
            block = appendActive(ctr + kCtrNeeBlocks) * (1u + fullSamples);
            uint choice = 0;
            if constexpr (kFill) addFillSpecAvgChoice(choice, preFlags, preCounters);
            p.neeBlocks[block] = make_uint4(slot, choice, 0u, 0u);
        }
        for (uint lightSample = 0; lightSample < (MULTI ? fullSamples : 1u); lightSample++)
        {
            float3 pickLi = mk3(0.f), pickDir = mk3(0.f); float pickDist = 0.f, pickSelPdf = 0.f, pickSolidPdf = 0.f;
            float weightSum = 0.f, pickWeight = 0.f; bool pickBsdfSampleable = true;
            uint pickLight = 0xFFFFFFFFu; bool pickLocal = false;
            // The candidate loop is a chain of dependent random gathers (proxy table -> counter, light record).  The light selection draws are
            // every 4th value of the stream, so the proxy lookups of the first 8 candidates are issued up front and their light records
            // prefetched into L2/L1 before the loop consumes them one by one.
            constexpr uint kPrefetch = 8;
            uint preLight[kPrefetch];
            {
                UniformSeq pre = uniformSG;
                #pragma unroll
                for (uint i = 0; i < kPrefetch; i++)
                {
                    preLight[i] = 0;
                    if (i < globalCount)
                    {
                        const float rnd = pre.next(); pre.next(); pre.next(); pre.next();
                        preLight[i] = __ldg(proxyIndices + min(uint(rnd * float(M)), M - 1));
                    }
                }
                #pragma unroll
                for (uint i = 0; i < kPrefetch; i++)
                    if (i < globalCount)
                    {
    #ifdef __CUDA_ARCH__    // (the host build of tests/emu/shade_host_emu.cu has no PTX)
                        asm volatile("prefetch.global.L1 [%0];" ::"l"(p.scene.lights + preLight[i]));
                        asm volatile("prefetch.global.L1 [%0];" ::"l"(proxyCounters + preLight[i]));
    #endif
                    }
            }
            #pragma unroll 1
            for (uint i = 0; i < candidateCount; i++)
            {
                const float rnd = uniformSG.next();
                uint lightIndex;
                switch (i)
                {   // static indexing keeps preLight[] in registers
                case 0: lightIndex = preLight[0]; break; case 1: lightIndex = preLight[1]; break; case 2: lightIndex = preLight[2]; break; case 3: lightIndex = preLight[3]; break;
                case 4: lightIndex = preLight[4]; break; case 5: lightIndex = preLight[5]; break; case 6: lightIndex = preLight[6]; break; case 7: lightIndex = preLight[7]; break;
                default: lightIndex = proxyIndices[min(uint(rnd * float(M)), M - 1)]; break;
                }
                float selectionPdf;
                const bool sampleIsLocal = NEEAT && i >= globalCount;
                if (sampleIsLocal) lightIndex = neeat::sampleLocal(p.na, tileAddress, rnd, selectionPdf);
                else selectionPdf = float(proxyCounters[lightIndex]) / float(M);
                const LightInfo li = p.scene.lights[lightIndex];
                const float r0 = uniformSG.next(), r1 = uniformSG.next();
                float3 lsPos = mk3(0.f), lsRadiance = mk3(0.f); float lsSolidPdf = 0.f; bool lsBsdfSampleable = true;
                if (ANALYTIC_LIGHTS && lightType(li) == kLightTypeSphere)
                {   // SphereLight::CalcSample (PolymorphicLight.hlsli:107-181): cone sampling of the visible cap; never found by BSDF rays
                    lsBsdfSampleable = false;
                    sampleSphereLight(li, p.scene, lightIndex, r0, r1, s.posW, lsPos, lsRadiance, lsSolidPdf);
                }
                else if (lightType(li) == kLightTypeTriangle)
                {   // TriangleLight::CalcSample (PolymorphicLight.hlsli:409-441)
                    TriLight tl; tl.decode(li);
                    const float sq = sqrtf(r0);
                    lsPos = offsetRayOrigin(tl.base + tl.e1 * (sq * (1 - r1)) + tl.e2 * (sq * r1), tl.normal);
                    const float3 toLight = lsPos - s.posW;
                    const float dist = sqrtf(fmaxf(2e-9f, dot3(toLight, toLight)));
                    const float cosTheta = dot3(tl.normal, -(toLight / dist));
                    if (cosTheta > 0.f) { lsSolidPdf = fminf(1e10f, pdfAreaToSolidAngle(fmaxf(2e-9f, 1.0f / tl.area), dist, cosTheta)); lsRadiance = tl.radiance; }
                }
                else if (lightType(li) == kLightTypeEnvQuad)
                {   // EnvironmentQuadLight::CalcSample (PolymorphicLight.hlsli:576-599), NEE_AT_SAMPLE_BAKED_ENVIRONMENT
                    const uint nodeX = li.direction1 >> 16, nodeY = li.direction1 & 0xFFFF, nodeDim = li.direction2 >> 16;
                    const float3 worldDir = rowVecTimes3x3(octEqualAreaToDir(mk2((float(nodeX) + r0) / float(nodeDim), (float(nodeY) + r1) / float(nodeDim))), p.c.envMap.Transform);
                    lsPos = s.posW + worldDir * kDistantLightDistance;
                    lsRadiance = unpackLightRadiance(li);
                    lsSolidPdf = float(nodeDim * nodeDim) / (4.0f * kPi);
                }
                const float pdf = lsSolidPdf * selectionPdf;
                const float3 Li = pdf > 0.f ? (lsRadiance / pdf) : mk3(0.f);
                const float3 surfToLight = lsPos - s.posW;
                const float dist = len3(surfToLight);
                const float3 dirToLight = surfToLight / fmaxf(dist, 1e-7f);
                const float wrsWeight = maxComp(Li) * bsdf.pdf(dirToLight);
                const float wrsRnd = uniformSG.next();
                weightSum += wrsWeight;
                if (wrsRnd < sat(wrsWeight / weightSum)) { pickLi = Li; pickDir = dirToLight; pickDist = dist; pickSelPdf = selectionPdf; pickSolidPdf = lsSolidPdf; pickWeight = wrsWeight; pickBsdfSampleable = lsBsdfSampleable; if (NEEAT) { pickLight = lightIndex; pickLocal = sampleIsLocal; } }
            }
            pickLi = pickLi * (1.0f / (pickWeight / weightSum));
            if (anyPositive(pickLi))
            {   // ProcessLightSample with visibility deferred to the shadow kernel
                const float fadeOut = (s.shadowNoLFadeout > 0) ? sat((dot3(pickDir, s.vertexN) - s.shadowNoLFadeout) / (2.0f * s.shadowNoLFadeout)) : 1.0f;
                // ComputeLightSelectionPdfs: the pdf the other sampler would have picked this light with, and how many candidates this sampler drew
                float otherPdf = 0.0f, thisCount = float(candidateCount);
                if constexpr (NEEAT)
                {
                    thisCount = float(globalCount);
                    if (pickLocal) { otherPdf = naGlobalLightPdf(p, pickLight); thisCount = float(localCount); }
                    else if (localCount != 0) otherPdf = neeat::sampleLocalPdf(p.na, tileAddress, pickLight);
                }
                const float wrsMIS = misBalance(pickSelPdf, otherPdf) / thisCount;             // without feedback all candidates come from the global table
                const float scatterPdfForDir = bsdf.pdf(pickDir);
                const float pathMIS = AMIS ? misApproxForLight(fullSamples, candidateCount, pickBsdfSampleable ? scatterPdfForDir : 0.0f)     // PathTracerNEE.hlsli:228-229
                                           : misBalance((pickSelPdf + otherPdf) * float(fullSamples) * pickSolidPdf, pickBsdfSampleable ? scatterPdfForDir : 0.0f);    // LightSampleableByBSDF
                const float3 Li = pickLi * (fadeOut * wrsMIS * pathMIS / float(fullSamples));
                const float4 bsdfThp = bsdf.eval(pickDir);
                float3 radiance = mk3(bsdfThp.x, bsdfThp.y, bsdfThp.z) * Li;
                const float radianceAvg = average(radiance);
                float specAvg = bsdfThp.w * average(Li);
                if (p.c.fireflyFilterThreshold != 0)
                {
                    const float k = newFireflyK(preFireflyK, pickSelPdf * pickSolidPdf, 1.0f);
                    const float thr = p.c.fireflyFilterThreshold * k;
                    radiance = radiance * ((radianceAvg > thr) ? (1.0f / radianceAvg * thr) : 1.0f);
                }
                radiance = radiance * preThp;
                specAvg *= average(preThp);
                if constexpr (NEEAT)
                {   // InsertFeedbackFromNEE's weight (un-filtered radiance x path throughput, biased towards globally improbable lights), inserted by the shadow kernel if visible
                    naFeedback = pickLight | (isSSC ? 0x80000000u : 0u);
                    naFeedbackWeight = __fdiv_rn(radianceAvg * average(preThp), powf(naGlobalLightPdf(p, pickLight), 0.65f));
                }
                const float faceSide = dot3(s.N, pickDir) >= 0 ? 1.0f : -1.0f;
                const float3 o = offsetRayOrigin(s.posW, s.faceN * faceSide);
                if constexpr (MULTI)
                {   // this sample's shadow record (long rays first, as appendShadowRecord) and its result, which k_nee_resolve adds if the shadow kernel marks it visible
                    const uint e = appendShadowRecordActive(p, ctr, pickDist * 0.9985f, neeShadowCapacity(p));
                    p.wf.shadowOriginTMax[e] = make_float4(o.x, o.y, o.z, pickDist * 0.9985f);
                    p.wf.shadowDirPath[e] = make_float4(pickDir.x, pickDir.y, pickDir.z, __uint_as_float(block));
                    p.wf.shadowRadiance[e] = make_uint2(lightSample, 0u);
                    p.neeBlocks[block + 1u + lightSample] = make_uint4(__float_as_uint(radiance.x), __float_as_uint(radiance.y), __float_as_uint(radiance.z), __float_as_uint(specAvg));
                }
                else
                {
                    out.emitShadow = true;
                    out.shadow.originTMax = make_float4(o.x, o.y, o.z, pickDist * 0.9985f);
                    out.shadow.dirPath = make_float4(pickDir.x, pickDir.y, pickDir.z, __uint_as_float(slot));
                    out.shadow.radiance = make_uint2(packHalf2Clamp(radiance.x, radiance.y), packHalf2Clamp(radiance.z, specAvg));   // NEEResult::AccumulateRadiance(0 + x)
                    if constexpr (kFill) addFillSpecAvgChoice(out.shadow.radiance.x, preFlags, preCounters);     // the specular average the shadow kernel adds with the radiance
                }
            }
        }
    }
    path.setMisInfo_RuRu(neeMis, path.ruRuCorrection());
    if (!scatterValid) path.setFlag(kPFActive, false);

    bool shouldTerminate = hasFinishedSurfaceBounces(p.c, path.vertexIndex() + 1, path.counter(kCtrDiffuseBounces));
    if (p.c.enableRussianRoulette)
    {   // HandleRussianRoulette (PathTracer.hlsli:182-208)
        const float rrVal = sqrtf(luminance(path.thp()));
        float prob = sat(0.85f - rrVal); prob = prob * prob;
        prob = sat(prob + fmaxf(0.0f, (float(path.vertexIndex()) / float(p.c.bounceCount) - 0.4f)));
        const bool finished = shouldTerminate;
        const float rrRnd = uniformSG.next();
        if constexpr (NEEAT)
        {   // had the light sample been visible, rrRnd is the feedback reservoir's number and roulette gets the next one: keep that outcome for the shadow kernel to publish
            if (out.emitShadow && p.na.temporalFeedbackRequired)
            {
                // (roulette runs - and, when it lets the path live, stores its correction - even on a path the bounce limit already ends: PathTracer.hlsli:756-760)
                const bool altRoulette = uniformSG.next() < prob, altTerminate = finished || altRoulette;
                out.naRecord = make_uint4(naFeedback, __float_as_uint(naFeedbackWeight), __float_as_uint(rrRnd),
                                          0x80000000u | (altTerminate ? 0x40000000u : 0u) | (altRoulette ? f32tof16(path.ruRuCorrection()) : f32tof16(1.0f / (1.0f - prob))));
            }
        }
        if (rrRnd < prob) shouldTerminate = true;
        else path.setMisInfo_RuRu(path.misInfo(), lp(1.0f / (1.0f - prob)));
    }
    else if constexpr (NEEAT)
    {
        if (out.emitShadow && p.na.temporalFeedbackRequired)
            out.naRecord = make_uint4(naFeedback, __float_as_uint(naFeedbackWeight), __float_as_uint(uniformSG.next()), 0x80000000u | (shouldTerminate ? 0x40000000u : 0u) | f32tof16(path.ruRuCorrection()));
    }
    if (shouldTerminate) path.setFlag(kPFTerminateAtNextBounce, true);
    out.continuePath = path.hasFlag(kPFActive);
}

} // namespace pt
