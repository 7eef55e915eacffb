// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of rtxpt_b200/csrc/debug_views.cuh (the pixel functions the debug-view kernels run) for tests/test_debug_views_port.py, which compares it with the oracle's
// restatement (oracle/pt_debug_views.h) on random surfaces and plane records.  Built by debug_views.mk.
#include "../../rtxpt_b200/csrc/debug_views.cuh"
#include <cstring>

using namespace pt;

static float kf(uint32_t w) { float f; std::memcpy(&f, &w, 4); return f; }

// in: count records of 28 words: barycentrics (2), faceN, vertexN, N, T, B (15), frontFacing, thin, diffuse (3), specular (3), roughness, metallic (f32), materialID (u32)
// out: count x 4 floats
extern "C" void debug_first_hit_emu(uint32_t view, const uint32_t* in, uint32_t count, float* out)
{
    for (uint32_t i = 0; i < count; i++, in += 28)
    {
        FirstHitDebugInputs d;
        d.barycentrics = mk2(kf(in[0]), kf(in[1]));
        float3* v[5] = { &d.faceN, &d.vertexN, &d.N, &d.T, &d.B };
        for (int k = 0; k < 5; k++) *v[k] = mk3(kf(in[2 + 3 * k]), kf(in[3 + 3 * k]), kf(in[4 + 3 * k]));
        d.frontFacing = in[17] != 0; d.thin = in[18] != 0;
        d.diffuse = mk3(kf(in[19]), kf(in[20]), kf(in[21])); d.specular = mk3(kf(in[22]), kf(in[23]), kf(in[24]));
        d.roughness = kf(in[25]); d.metallic = kf(in[26]); d.materialID = in[27];
        const float4 c = firstHitDebugColor(view, d);
        out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.z; out[4 * i + 3] = c.w;
    }
}

// the realtime buffers in the library's layout: planes in GenericTS addressing, header [4][H][W], stable radiance RGBA16F
struct HostBuffers
{
    const RtxptStablePlane* planes; const uint32_t* header; const uint16_t* radiance; uint W, H, lineStride, planeStride;
    __host__ __device__ uint branchID(uint x, uint y, uint plane) const { return header[(size_t(plane) * H + y) * W + x]; }
    __host__ __device__ RtxptStablePlane plane(uint x, uint y, uint plane) const
    {
        const uint xi = x & 7u, yi = y & 7u;
        return planes[(x - xi) * 8u + (y - yi) * lineStride + morton(xi, yi) + plane * planeStride];
    }
    __host__ __device__ uint dominantIndex(uint x, uint y) const { return header[(size_t(3) * H + y) * W + x] & 3u; }
    __host__ __device__ float3 stableRadiance(uint x, uint y) const { const uint16_t* r = radiance + (size_t(y) * W + x) * 4; return mk3(f16tof32(r[0]), f16tof32(r[1]), f16tof32(r[2])); }
    __host__ __device__ static uint morton(uint x, uint y) { uint m = 0; for (uint b = 0; b < 3; b++) m |= (((x >> b) & 1u) << (2 * b)) | (((y >> b) & 1u) << (2 * b + 1)); return m; }
};

// out: W x H x 4 floats, 0 where nothing is drawn
extern "C" void debug_stable_planes_emu(uint32_t view, int32_t dbgPlaneIndex, uint32_t W, uint32_t H, uint32_t lineStride, uint32_t planeStride, const RtxptStablePlane* planes,
                                        const uint32_t* header, const uint16_t* stableRadiance, float* out)
{
    const HostBuffers b{ planes, header, stableRadiance, W, H, lineStride, planeStride };
    for (uint y = 0; y < H; y++)
        for (uint x = 0; x < W; x++)
        {
            float4 c = stablePlaneDebugPixel(view, dbgPlaneIndex, x, y, W, H, b);
            if (!(c.w > 0.0f)) c = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            float* o = out + (size_t(y) * W + x) * 4; o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = c.w;
        }
}

// the colour functions alone, in the records of oracle/ref_kat_debug_main.cpp (tests/golden/debug_view_golden.npz): per record op, a, b, c -> 3 words
extern "C" void debug_pixel_funcs_emu(const uint32_t* in, uint32_t count, uint32_t* out)
{
    for (uint32_t i = 0; i < count; i++, in += 4, out += 3)
    {
        const uint32_t op = in[0], a = in[1], b = in[2], c = in[3];
        if (op == 3) { stablePlaneFourWaySplitCoord(int(a), b & 0xFFFFu, b >> 16, c & 0xFFFFu, c >> 16, out[0], out[1], out[2]); continue; }
        float3 r;
        if (op == 0) r = colorFromHash(a);
        else if (op == 1) r = gradientHeatMap(kf(a));
        else if (op == 2) r = stablePlaneDebugVizColor(a);
        else r = dbgShowNormalSRGB(mk3(kf(a), kf(b), kf(c)));
        out[0] = floatBits(r.x); out[1] = floatBits(r.y); out[2] = floatBits(r.z);
    }
}
