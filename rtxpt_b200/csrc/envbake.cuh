// envbake.cuh - the environment-map baking path (SURVEY §8f row 3; replaces EnvMapBaker's BaseLayerCS / MIPReduceCS, Rtxpt/Lighting/Distant/EnvMapBaker.hlsl:64-356 and
// EnvMapBaker.cpp:425-600): an equirectangular or cube source plus up to 16 directional lights baked into the RGBA16F cube the path tracer samples, and its MIP chain with
// solid-angle weights.  Pass bodies are __host__ __device__ (kernels: envbake_kernels.cu; host build for the CPU parity test: tests/emu).  Not built: the procedural sky, the
// BC6U compression of the result (RTXPT's default; this is its compression quality 0), seamless cross-face filtering of a cube source (taps clamp to the face).
#pragma once
#include "device_math.cuh"

namespace pt { namespace envbake {

struct DirectionalLight { float colorIntensity[4]; float direction[3]; float angularSize; };     // EMB_DirectionalLight: colour, W/sr, incoming direction, radians
struct Params
{
    uint cubeDim, sourceType, sourceWidth, sourceHeight;    // sourceType: 0 none, 1 equirectangular, 2 cube (+x -x +y -y +z -z)
    const float* source;                                    // RGBA32F
    float scaleColor[3]; uint lightCount;
    DirectionalLight lights[16];
    float* mips[16];                                        // MIP m: 6 faces of (cubeDim >> m)^2 RGBA32F texels holding fp16 values
};

PT_HD float lpf(float v) { return f16tof32(f32tof16(v)); }
PT_HD float3 cubemapDirectionFor(uint face, float u, float v)
{
    const float cx = (u * 2.0f) - 1, cy = 1 - (v * 2.0f);
    const float l = sqrtf(cx * cx + cy * cy + 1);
    float3 d = mk3(0.f);
    switch (face)
    {
    case 0: d = mk3(1, cy, -cx); break;  case 1: d = mk3(-1, cy, cx); break;
    case 2: d = mk3(cx, 1, -cy); break;  case 3: d = mk3(cx, -1, cy); break;
    case 4: d = mk3(cx, cy, 1); break;   case 5: d = mk3(-cx, cy, -1); break;
    }
    return d * (1 / l);
}
PT_HD float sphereQuadrantArea(float x, float y) { return atan2f(x * y, sqrtf(x * x + y * y + 1)); }
PT_HD float4 texelSolidAngle4(float cubeDim, uint tlx, uint tly)
{
    const float iDim = 1.0f / cubeDim;
    const float s = ((float(tlx) + 0.5f) * 2 * iDim) - 1, t = ((float(tly) + 0.5f) * 2 * iDim) - 1;
    const float x0 = s - iDim, y0 = t - iDim, x1 = s + iDim, y1 = t + iDim, x2 = s + iDim * 3, y2 = t + iDim * 3;
    const float a00 = sphereQuadrantArea(x0, y0), a01 = sphereQuadrantArea(x0, y1), a10 = sphereQuadrantArea(x1, y0), a11 = sphereQuadrantArea(x1, y1), a20 = sphereQuadrantArea(x2, y0),
                a21 = sphereQuadrantArea(x2, y1), a02 = sphereQuadrantArea(x0, y2), a12 = sphereQuadrantArea(x1, y2), a22 = sphereQuadrantArea(x2, y2);
    return make_float4(fmaxf(1e-6f, fabsf(a00 - a01 - a10 + a11)), fmaxf(1e-6f, fabsf(a01 - a02 - a11 + a12)), fmaxf(1e-6f, fabsf(a10 - a11 - a20 + a21)), fmaxf(1e-6f, fabsf(a11 - a12 - a21 + a22)));
}
PT_HD int wrapi(int x, int n) { return ((x % n) + n) % n; }
PT_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
PT_HD float3 sampleBilinear(const float* img, int W, int H, float u, float v, bool wrapU)
{
    const float tx = u * float(W) - 0.5f, ty = v * float(H) - 0.5f, fx = floorf(tx), fy = floorf(ty), wx = tx - fx, wy = ty - fy;
    const int x0 = wrapU ? wrapi(int(fx), W) : clampi(int(fx), 0, W - 1), x1 = wrapU ? wrapi(int(fx) + 1, W) : clampi(int(fx) + 1, 0, W - 1), y0 = clampi(int(fy), 0, H - 1), y1 = clampi(int(fy) + 1, 0, H - 1);
    const float* a = img + (size_t(y0) * W + x0) * 4; const float* b = img + (size_t(y0) * W + x1) * 4; const float* c = img + (size_t(y1) * W + x0) * 4; const float* d = img + (size_t(y1) * W + x1) * 4;
    return (mk3(a[0], a[1], a[2]) * (1 - wx) + mk3(b[0], b[1], b[2]) * wx) * (1 - wy) + (mk3(c[0], c[1], c[2]) * (1 - wx) + mk3(d[0], d[1], d[2]) * wx) * wy;
}
PT_HD float3 sampleSource(const Params& p, uint px, uint py, uint face)
{
    const float3 dir = cubemapDirectionFor(face, (float(px) + 0.5f) / float(p.cubeDim), (float(py) + 0.5f) / float(p.cubeDim));
    if (p.sourceType == 1)
    {   // world_to_latlong_map (MathHelpers.hlsli:92-99); bilinear, wrap in u, clamp in v (EnvMapBaker.cpp:156-159)
        const float3 n = norm3(dir);
        return sampleBilinear(p.source, int(p.sourceWidth), int(p.sourceHeight), atan2f(n.x, -n.z) * 0.15915494309189535f + 0.5f, acosf(n.y) * 0.3183098861837907f, true);
    }
    if (p.sourceType == 2)
    {
        const float ax = fabsf(dir.x), ay = fabsf(dir.y), az = fabsf(dir.z);
        uint f; float cx, cy;
        if (ax >= ay && ax >= az) { f = dir.x > 0 ? 0u : 1u; cx = dir.x > 0 ? -dir.z / ax : dir.z / ax; cy = dir.y / ax; }
        else if (ay >= az) { f = dir.y > 0 ? 2u : 3u; cx = dir.x / ay; cy = dir.y > 0 ? -dir.z / ay : dir.z / ay; }
        else { f = dir.z > 0 ? 4u : 5u; cx = dir.z > 0 ? dir.x / az : -dir.x / az; cy = dir.y / az; }
        return sampleBilinear(p.source + size_t(f) * p.sourceWidth * p.sourceWidth * 4, int(p.sourceWidth), int(p.sourceWidth), (cx + 1) * 0.5f, (1 - cy) * 0.5f, false);
    }
    return mk3(0.f);
}
// anti-aliased coverage of the light's cone by the texel (four corners of a 1.1-texel footprint), ^4 "to roughly account for tone mapping"
PT_HD float3 lightContribution(const Params& p, uint px, uint py, uint face, const DirectionalLight& light)
{
    const float fade = 1.1f, dim = float(p.cubeDim);
    const float3 toLight = mk3(-light.direction[0], -light.direction[1], -light.direction[2]);
    float dotMin = 1e30f, dotMax = -1e30f;
    #pragma unroll
    for (int k = 0; k < 4; k++)
    {
        const float ox = (k & 1) ? fade : -fade, oy = (k & 2) ? fade : -fade;
        const float c = dot3(toLight, cubemapDirectionFor(face, (float(px) + 0.5f + 0.5f * ox) / dim, (float(py) + 0.5f + 0.5f * oy) / dim));
        dotMin = fminf(dotMin, c); dotMax = fmaxf(dotMax, c);
    }
    const float angleMin = acosf(clampf(dotMax, -1.0f, 1.0f)), angleMax = acosf(clampf(dotMin, -1.0f, 1.0f));
    float coverage = sat(((light.angularSize * 0.5f) - angleMin) / (angleMax - angleMin + 1e-24f));
    coverage = powf(coverage, 4.0f);
    const float lightSolidAngle = 2 * kPi * (1 - cosf(light.angularSize * 0.5f));
    return mk3(light.colorIntensity[0], light.colorIntensity[1], light.colorIntensity[2]) * (coverage * (light.colorIntensity[3] / lightSolidAngle));
}
PT_HD float4 generateTexel(const Params& p, uint px, uint py, uint face)
{
    float3 c = sampleSource(p, px, py, face);
    for (uint i = 0; i < p.lightCount; i++) c = c + lightContribution(p, px, py, face, p.lights[i]);
    c = c * mk3(p.scaleColor[0], p.scaleColor[1], p.scaleColor[2]);
    return make_float4(lpf(clampf(c.x, 0.0f, 65504.0f)), lpf(clampf(c.y, 0.0f, 65504.0f)), lpf(clampf(c.z, 0.0f, 65504.0f)), 1.0f);
}
PT_HD float* texelAt(const Params& p, uint mip, uint face, uint x, uint y) { const uint n = p.cubeDim >> mip; return p.mips[mip] + ((size_t(face) * n + y) * n + x) * 4; }
PT_HD void storeTexel(float* d, float4 v) { d[0] = lpf(v.x); d[1] = lpf(v.y); d[2] = lpf(v.z); d[3] = lpf(v.w); }
PT_HD float4 weightedAverage(float4 a, float4 b, float4 c, float4 d, float4 w)
{
    const float wsum = w.x + w.y + w.z + w.w;
    return make_float4((a.x * w.x + b.x * w.y + c.x * w.z + d.x * w.w) / wsum, (a.y * w.x + b.y * w.y + c.y * w.z + d.y * w.w) / wsum, (a.z * w.x + b.z * w.y + c.z * w.z + d.z * w.w) / wsum,
                       (a.w * w.x + b.w * w.y + c.w * w.z + d.w * w.w) / wsum);
}
// BaseLayerCS: thread (x, y, face) over the half-resolution grid writes four MIP 0 texels and their solid-angle-weighted MIP 1 texel
PT_HD void baseLayerTexel(const Params& p, uint x, uint y, uint face, bool hasMip1)
{
    const float4 w = texelSolidAngle4(float(p.cubeDim), x * 2, y * 2);
    const float4 e00 = generateTexel(p, x * 2, y * 2, face), e01 = generateTexel(p, x * 2, y * 2 + 1, face), e10 = generateTexel(p, x * 2 + 1, y * 2, face), e11 = generateTexel(p, x * 2 + 1, y * 2 + 1, face);
    storeTexel(texelAt(p, 0, face, x * 2, y * 2), e00); storeTexel(texelAt(p, 0, face, x * 2, y * 2 + 1), e01); storeTexel(texelAt(p, 0, face, x * 2 + 1, y * 2), e10); storeTexel(texelAt(p, 0, face, x * 2 + 1, y * 2 + 1), e11);
    if (hasMip1) storeTexel(texelAt(p, 1, face, x, y), weightedAverage(e00, e01, e10, e11, w));
}
// MIPReduceCS: texel (x, y, face) of MIP m from the 2x2 of MIP m - 1
PT_HD void mipReduceTexel(const Params& p, uint mip, uint x, uint y, uint face)
{
    const uint n = p.cubeDim >> mip;
    const float4 w = texelSolidAngle4(float(n * 2), x * 2, y * 2);
    const float* a = texelAt(p, mip - 1, face, x * 2, y * 2); const float* b = texelAt(p, mip - 1, face, x * 2, y * 2 + 1); const float* c = texelAt(p, mip - 1, face, x * 2 + 1, y * 2); const float* d = texelAt(p, mip - 1, face, x * 2 + 1, y * 2 + 1);
    storeTexel(texelAt(p, mip, face, x, y), weightedAverage(make_float4(a[0], a[1], a[2], a[3]), make_float4(b[0], b[1], b[2], b[3]), make_float4(c[0], c[1], c[2], c[3]), make_float4(d[0], d[1], d[2], d[3]), w));
}

// ---- importance / radiance map of a re-baked cube (BuildMIPDescentImportanceMapCS, EnvMapImportanceSamplingBaker.hlsl:56-90, + the 2x2 box MIP chain after it) ----------------
// A second implementation of LightBaker::buildEnvRadianceMap (lights_bake.cpp), on purpose: the host one serves the scene upload, this one rtxpt_b200_update_env_map.  Every
// operation follows the host's order (face selection, 8-bit bilinear weights, per-face clamp, summation order, fp16 rounding), so the host build of these bodies equals the host map
// bit for bit (tests/test_env_update.py).  On the GPU the cos / sin of the octahedral mapping come from libdevice and the host's from the C library; neither is correctly
// rounded, so the two maps differ in a small share of texels and the upload keeps the host map (the light tables of an upload stay those the oracle holds bit for bit).
constexpr uint kImportanceDim = 1024, kImportanceMips = 11, kImportanceSamples = 4;       // EMISB_IMPORTANCE_MAP_DIM, EMISB_IMPORTANCE_SAMPLES_PER_PIXEL^2 = 16 taps
struct ImportanceParams
{
    const float* cube; uint faceSize;                       // MIP 0 of the bake: 6 faces of faceSize^2 RGBA32F texels
    float* mips[kImportanceMips];                           // MIP m: (1024 >> m)^2 RGBA32F texels holding fp16 values (.a = importance)
};
PT_HD float3 octEqualAreaToDirHD(float u, float v)      // oct_to_ndir_equal_area_unorm with the host's constant and sign function
{
    const float px = u * 2.f - 1.f, py = v * 2.f - 1.f;
    const float d = 1.f - (fabsf(px) + fabsf(py));
    const float r = 1.f - fabsf(d);
    const float phi = (r > 0.f) ? ((fabsf(py) - fabsf(px)) / r + 1.f) * 0.78539816339744830961f : 0.f;
    const float f = r * sqrtf(2.f - r * r);
    const float sx = (px > 0.f) ? 1.f : ((px < 0.f) ? -1.f : 0.f), sy = (py > 0.f) ? 1.f : ((py < 0.f) ? -1.f : 0.f), sd = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
    return mk3(f * sx * cosf(phi), f * sy * sinf(phi), sd * (1.f - r * r));
}
PT_HD float q8(float a) { return floorf(a * 256.0f + 0.5f) * (1.0f / 256.0f); }        // 8 fractional bits, like the texture units
PT_HD float3 cubeTexel(const ImportanceParams& p, uint face, int x, int y)
{
    const int n = int(p.faceSize);
    x = clampi(x, 0, n - 1); y = clampi(y, 0, n - 1);
    const float* t = p.cube + ((size_t(face) * n + y) * n + x) * 4;
    return mk3(t[0], t[1], t[2]);
}
PT_HD float3 sampleCubeMip0(const ImportanceParams& p, float3 v)
{
    const float ax = fabsf(v.x), ay = fabsf(v.y), az = fabsf(v.z);
    float m, s, t; uint face;
    if (ax >= ay && ax >= az) { m = ax; if (v.x >= 0) { face = 0; s = -v.z; t = -v.y; } else { face = 1; s = v.z; t = -v.y; } }
    else if (ay >= az)        { m = ay; if (v.y >= 0) { face = 2; s = v.x; t = v.z; }  else { face = 3; s = v.x; t = -v.z; } }
    else                      { m = az; if (v.z >= 0) { face = 4; s = v.x; t = -v.y; } else { face = 5; s = -v.x; t = -v.y; } }
    const float n = float(p.faceSize);
    const float x = (s / m + 1.0f) * 0.5f * n - 0.5f, y = (t / m + 1.0f) * 0.5f * n - 0.5f;
    const float fx = floorf(x), fy = floorf(y);
    const float wx = q8(x - fx), wy = q8(y - fy);
    const int ix = int(fx), iy = int(fy);
    const float3 a = cubeTexel(p, face, ix, iy) * (1 - wx) + cubeTexel(p, face, ix + 1, iy) * wx;
    const float3 b = cubeTexel(p, face, ix, iy + 1) * (1 - wx) + cubeTexel(p, face, ix + 1, iy + 1) * wx;
    return a * (1 - wy) + b * wy;
}
// texel (px, py) of MIP 0: 4 x 4 taps, radiance and (luminance + average) / 2 importance
PT_HD void importanceTexel(const ImportanceParams& p, uint px, uint py)
{
    const uint N = kImportanceDim, S = kImportanceSamples;
    const float inv = 1.0f / float(S * S);
    float L = 0.f; float3 R = mk3(0.f);
    for (uint y = 0; y < S; y++)
        for (uint x = 0; x < S; x++)
        {
            const float3 dir = octEqualAreaToDirHD((float(px * S + x) + 0.5f) / float(N * S), (float(py * S + y) + 0.5f) / float(N * S));
            const float3 rad = sampleCubeMip0(p, dir);
            const float lum = rad.x * 0.2126f + rad.y * 0.7152f + rad.z * 0.0722f, avg = (rad.x + rad.y + rad.z) / 3.0f;
            L += (lum + avg) * 0.5f;
            R = R + rad;
        }
    float* o = p.mips[0] + (size_t(py) * N + px) * 4;
    o[0] = lpf(R.x * inv); o[1] = lpf(R.y * inv); o[2] = lpf(R.z * inv); o[3] = lpf(L * inv);
}
// texel (x, y) of MIP m >= 1: the 2x2 box of MIP m - 1 (donut's MipMapGenPass, MODE_COLOR)
PT_HD void importanceReduceTexel(const ImportanceParams& p, uint mip, uint x, uint y)
{
    const uint n = kImportanceDim >> mip, pn = kImportanceDim >> (mip - 1);
    const float* src = p.mips[mip - 1];
    for (uint c = 0; c < 4; c++)
    {
        const float s = src[(size_t(2 * y) * pn + 2 * x) * 4 + c] + src[(size_t(2 * y) * pn + 2 * x + 1) * 4 + c] + src[(size_t(2 * y + 1) * pn + 2 * x) * 4 + c] + src[(size_t(2 * y + 1) * pn + 2 * x + 1) * 4 + c];
        p.mips[mip][(size_t(y) * n + x) * 4 + c] = lpf(s * 0.25f);
    }
}

} } // namespace pt::envbake
