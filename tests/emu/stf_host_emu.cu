// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of rtxpt_b200/csrc/stf.cuh (the sample-position code every STF material fetch of the shade kernels runs) for tests/test_stf_port.py: the same records as
// oracle/ref_kat_stf_main.cpp takes and writes, so that the two can be compared word for word (tests/golden/stf_golden.npz).  Built by stf.mk.
#include "../../rtxpt_b200/csrc/stf.cuh"
#include <cstring>
#include <algorithm>

using namespace pt;

static float kf(uint32_t w) { float f; std::memcpy(&f, &w, 4); return f; }
static uint32_t kw(float f) { uint32_t w; std::memcpy(&w, &f, 4); return w; }

// the texel a wrap or clamp sampler returns at a texel centre of an integer level, named (x, y, level, 1) as the reference driver's texture does
static float4 texelAt(uint w, uint h, float2 pos, uint level, uint addressMode)
{
    const uint lw = std::max(1u, w >> level), lh = std::max(1u, h >> level);
    long x = long(floorf(pos.x * float(lw))), y = long(floorf(pos.y * float(lh)));
    if (addressMode == kStfAddressClamp) { x = std::min(std::max(x, 0L), long(lw) - 1); y = std::min(std::max(y, 0L), long(lh) - 1); }
    else { x = ((x % long(lw)) + long(lw)) % long(lw); y = ((y % long(lh)) + long(lh)) % long(lh); }
    return make_float4(float(x), float(y), float(level), 1.0f);
}

// in: count records of 28 words, out: count x (4 x 11 + 10) words (see ref_kat_stf_main.cpp)
extern "C" void stf_emu_run(const uint32_t* in, uint32_t count, uint32_t* out)
{
    for (uint32_t c = 0; c < count; c++, in += 28)
    {
        StfState s;
        s.u = make_float4(kf(in[7]), kf(in[8]), kf(in[9]), kf(in[10]));
        s.filterType = in[3]; s.sigma = kf(in[4]); s.reseedOnSample = in[6] != 0;
        float lastX = 0.0f; uint lastW = 1;
        for (int f = 0; f < 4; f++)
        {
            const float2 uv = make_float2(kf(in[11 + 3 * f]), kf(in[12 + 3 * f]));
            const StfSamplePos p = stfTexture2DSamplePos(s, in[0], in[1], in[2], uv, kf(in[13 + 3 * f]));
            const float4 v = texelAt(in[0], in[1], p.uv, p.lod, in[5]);
            *out++ = kw(p.uv.x); *out++ = kw(p.uv.y); *out++ = p.lod;
            *out++ = kw(v.x); *out++ = kw(v.y); *out++ = kw(v.z); *out++ = kw(v.w);
            *out++ = kw(s.u.x); *out++ = kw(s.u.y); *out++ = kw(s.u.z); *out++ = kw(s.u.w);
            lastX = uv.x; lastW = std::max(1u, in[0] >> p.lod);
        }
        for (uint mode = 1; mode <= 5; mode++)
        {
            bool isBorder = false;
            *out++ = kw(stfApplyAddressingMode1D(lastX, lastW, mode, isBorder)); *out++ = isBorder ? 1u : 0u;
        }
    }
}

// the vertex's u as loadSurface draws it
extern "C" void stf_emu_vertex_random(uint32_t packedPixel, uint32_t vertexIndex, uint32_t sampleIndex, float* out4)
{
    const float4 u = stfVertexRandom(packedPixel, vertexIndex, sampleIndex);
    out4[0] = u.x; out4[1] = u.y; out4[2] = u.z; out4[3] = u.w;
}
