// ORACLE/_ref — TEST INFRASTRUCTURE.  Known-answer generator for the debug-view colour functions: the UNMODIFIED reference functions streamed behind ref_hlsl_shim.h by
// ref_debug_tu.sh.  This file is read twice: first with DEBUG_KAT_STANDINS for what the functions need beyond the shim, then, after them, for the driver.
//   stdin:  per record 4 words: op, a, b, c
//     op 0: ColorFromHash(a)                                 op 1: GradientHeatMap(asfloat(a))              op 2: StablePlaneDebugVizColor(a)
//     op 3: StablePlaneDebugVizFourWaySplitCoord(int(a), pixel (b & 0xFFFF, b >> 16), screen (c & 0xFFFF, c >> 16))    op 4: DbgShowNormalSRGB(asfloat(a, b, c))
//   stdout: per record 3 words: the float3 (ops 0-2, 4) or uint3 (op 3) result
#ifdef DEBUG_KAT_STANDINS
#include <cstdio>
#include <cstdint>
#include <vector>
// (the shim has everything the functions use)
#else
int main()
{
    std::vector<uint32_t> in; uint32_t w;
    while (std::fread(&w, 4, 1, stdin) == 1) in.push_back(w);
    for (size_t i = 0; i + 4 <= in.size(); i += 4)
    {
        const uint32_t op = in[i], a = in[i + 1], b = in[i + 2], c = in[i + 3];
        uint32_t out[3] = { 0, 0, 0 };
        if (op == 3)
        {
            const uint3 r = StablePlaneDebugVizFourWaySplitCoord(int(a), uint2(b & 0xFFFFu, b >> 16), uint2(c & 0xFFFFu, c >> 16));
            out[0] = r.x; out[1] = r.y; out[2] = r.z;
        }
        else
        {
            float3 r;
            if (op == 0) r = ColorFromHash(a);
            else if (op == 1) r = GradientHeatMap(asfloat(a));
            else if (op == 2) r = StablePlaneDebugVizColor(a);
            else r = DbgShowNormalSRGB(float3(asfloat(a), asfloat(b), asfloat(c)));
            out[0] = asuint(r.x); out[1] = asuint(r.y); out[2] = asuint(r.z);
        }
        std::fwrite(out, 4, 3, stdout);
    }
    return 0;
}
#endif
