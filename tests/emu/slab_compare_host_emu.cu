// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so, never loaded by rtxpt_b200/.
// Host build of the traversal's node step (rtxpt_b200/csrc/traverse.cuh: nodeHitMask, the same source Traverser::run inlines) next to the formulation it replaced, which lives
// only here as the reference: float min / max chains for the slab compare and a per-child extract / shift / select for the hit word.  tests/test_slab_compare_port.py runs both
// over every (node, ray) pair of a built tree; the two hit words have to be equal.  Built by slab_compare.mk.
#include "../../rtxpt_b200/csrc/traverse.cuh"
#include <cmath>
#include <cstdint>

using namespace pt;

// the node step as it was before the integer compare: t values computed exactly as nodeHitMask computes them, compared with fmaxf / fminf
static uint referenceHitMask(const uint4 n0, const uint4 n1, const uint4 n2, const uint4 n3, const uint4 n4, float3 org, float idx, float idy, float idz, uint octinv, float tMin, float bestT)
{
    const uint octinv4 = octinv * 0x01010101u;
    const bool negx = !(octinv & 4u), negy = !(octinv & 2u), negz = !(octinv & 1u);
    const float px = bitsToFloat(n0.x), py = bitsToFloat(n0.y), pz = bitsToFloat(n0.z);
    const float sx15 = bitsToFloat(((n0.w & 0xFFu) + 15u) << 23), sy15 = bitsToFloat((((n0.w >> 8) & 0xFFu) + 15u) << 23), sz15 = bitsToFloat((((n0.w >> 16) & 0xFFu) + 15u) << 23);
    const float Ax15 = sx15 * idx, Ay15 = sy15 * idy, Az15 = sz15 * idz;
    const float Ax = (PT_I2F_AXES > 0) ? Ax15 * (1.0f / 32768.0f) : Ax15, Ay = (PT_I2F_AXES > 1) ? Ay15 * (1.0f / 32768.0f) : Ay15, Az = (PT_I2F_AXES > 2) ? Az15 * (1.0f / 32768.0f) : Az15;
    const float ox = (px - org.x) * idx, oy = (py - org.y) * idy, oz = (pz - org.z) * idz;
    const float Ox = (PT_I2F_AXES > 0) ? ox : ox - Ax, Oy = (PT_I2F_AXES > 1) ? oy : oy - Ay, Oz = (PT_I2F_AXES > 2) ? oz : oz - Az;
    const float kLo = 1.0f - 6.0e-7f, kHi = 1.0f + 6.0e-7f, kPad = 4.8e-7f;
    const float Anx = Ax * kLo, Any = Ay * kLo, Anz = Az * kLo, Afx = Ax * kHi, Afy = Ay * kHi, Afz = Az * kHi;
    const float Onx = fmaf(Ox, kLo, -fabsf(Ax15) * kPad), Ony = fmaf(Oy, kLo, -fabsf(Ay15) * kPad), Onz = fmaf(Oz, kLo, -fabsf(Az15) * kPad);
    const float Ofx = fmaf(Ox, kHi, fabsf(Ax15) * kPad), Ofy = fmaf(Oy, kHi, fabsf(Ay15) * kPad), Ofz = fmaf(Oz, kHi, fabsf(Az15) * kPad);
    uint hitmask = 0;
    for (int half = 0; half < 2; half++)
    {
        const uint meta4 = half ? n1.w : n1.z;
        const uint isInner4 = (meta4 & (meta4 << 1)) & 0x10101010u;
        const uint innerMask4 = (isInner4 >> 4) * 0xFFu;
        const uint bitIndex4 = (meta4 ^ (octinv4 & innerMask4)) & 0x1F1F1F1Fu;
        const uint childBits4 = (meta4 >> 5) & 0x07070707u;
        const uint qlox = half ? n2.y : n2.x, qloy = half ? n2.w : n2.z, qloz = half ? n3.y : n3.x;
        const uint qhix = half ? n3.w : n3.z, qhiy = half ? n4.y : n4.x, qhiz = half ? n4.w : n4.z;
        const uint nearx = negx ? qhix : qlox, farx = negx ? qlox : qhix;
        const uint neary = negy ? qhiy : qloy, fary = negy ? qloy : qhiy;
        const uint nearz = negz ? qhiz : qloz, farz = negz ? qloz : qhiz;
        for (int j = 0; j < 4; j++)
        {
            const float t0x = fmaf(byteToCoord<(PT_I2F_AXES > 0)>(nearx, j, 0), Anx, Onx), t1x = fmaf(byteToCoord<(PT_I2F_AXES > 0)>(farx, j, 0), Afx, Ofx);
            const float t0y = fmaf(byteToCoord<(PT_I2F_AXES > 1)>(neary, j, 0), Any, Ony), t1y = fmaf(byteToCoord<(PT_I2F_AXES > 1)>(fary, j, 0), Afy, Ofy);
            const float t0z = fmaf(byteToCoord<(PT_I2F_AXES > 2)>(nearz, j, 0), Anz, Onz), t1z = fmaf(byteToCoord<(PT_I2F_AXES > 2)>(farz, j, 0), Afz, Ofz);
            const float cmin = fmaxf(fmaxf(t0x, t0y), fmaxf(t0z, tMin));
            const float cmax = fminf(fminf(t1x, t1y), fminf(t1z, bestT));
            if (cmin <= cmax)
                hitmask |= ((childBits4 >> (8 * j)) & 0xFFu) << ((bitIndex4 >> (8 * j)) & 0xFFu);
        }
    }
    return hitmask;
}

// nodes: nodeCount x 20 words; rays: rayCount x 8 floats (origin, tMin, direction, tMax).  tMinZero != 0 runs the wavefront's instantiation (the rays' tMin must be 0), else the
// general one.  Returns the number of (node, ray) pairs whose hit words differ; firstMismatch = { node, ray, reference word, new word } of the first one in node order;
// *pairsWithHits counts the pairs with a non-zero reference word.
extern "C" uint64_t emu_slab_compare(const uint32_t* nodes, uint32_t nodeCount, const float* rays, uint32_t rayCount, int tMinZero, uint32_t* firstMismatch, uint64_t* pairsWithHits)
{
    uint64_t bad = 0, hits = 0;
    uint32_t firstNode = 0xFFFFFFFFu;
    #pragma omp parallel for schedule(static) reduction(+ : bad, hits)
    for (int64_t ni = 0; ni < int64_t(nodeCount); ni++)
    {
        const uint4* np = reinterpret_cast<const uint4*>(nodes + size_t(ni) * 20);
        for (uint32_t r = 0; r < rayCount; r++)
        {
            const float* q = rays + size_t(r) * 8;
            const float3 o = mk3(q[0], q[1], q[2]), d = mk3(q[4], q[5], q[6]);
            // the ray constants of Traverser::init (the host has no __fdividef: an IEEE quotient stands in, both formulations get the same one)
            const float eps = 1.0e-20f;
            const float idx = 1.0f / (fabsf(d.x) > eps ? d.x : copysignf(eps, d.x)), idy = 1.0f / (fabsf(d.y) > eps ? d.y : copysignf(eps, d.y)), idz = 1.0f / (fabsf(d.z) > eps ? d.z : copysignf(eps, d.z));
            const uint octinv = 7u - ((d.x < 0.0f ? 4u : 0u) | (d.y < 0.0f ? 2u : 0u) | (d.z < 0.0f ? 1u : 0u));
            const uint want = referenceHitMask(np[0], np[1], np[2], np[3], np[4], o, idx, idy, idz, octinv, q[3], q[7]);
            const uint got = tMinZero ? nodeHitMask<true>(np[0], np[1], np[2], np[3], np[4], o, idx, idy, idz, octinv, q[3], q[7], 0)
                                      : nodeHitMask<false>(np[0], np[1], np[2], np[3], np[4], o, idx, idy, idz, octinv, q[3], q[7], 0);
            hits += want != 0;
            if (want != got)
            {
                bad++;
                #pragma omp critical
                if (uint32_t(ni) < firstNode) { firstNode = uint32_t(ni); firstMismatch[0] = uint32_t(ni); firstMismatch[1] = r; firstMismatch[2] = want; firstMismatch[3] = got; }
            }
        }
    }
    *pairsWithHits = hits;
    return bad;
}
