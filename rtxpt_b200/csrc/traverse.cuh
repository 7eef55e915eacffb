// traverse.cuh — software ray queries: CWBVH8 traversal + watertight ray/triangle test + any-hit alpha test.
// Replaces what the reference delegates to RT cores through RayQuery::TraceRayInline:
//   Bridge::traceScatterRay  (Rtxpt/Shaders/PathTracerBridgeDonut.hlsli:1029-1055)  -> traceRay<false>
//   Bridge::traceVisibilityRay (…:993-1027, RAY_FLAG_ACCEPT_FIRST_HIT_AND_END_SEARCH)  -> traceRay<true>
//   AlphaTestImpl (…:929-971), AlphaTestVisibilityRay ExcludeFromNEE (…:980-989)
// Algorithms: Ylitie/Karras/Laine HPG 2017 (node-group / triangle-group stack, octant-ordered hit masks);
//             Woop/Benthin/Wald JCGT 2013 (watertight test; fp64 fallback when an edge function is exactly zero).
// Conventions shared with the oracle so hit records are bit-identical: no FMA contraction in the triangle test, t = T/det,
// (u,v) = (V/det, W/det), accept tMin < t < tMax, equal-t ties go to the smaller global triangle id.
#pragma once
#include "device_math.cuh"
#include "scene_device.cuh"
#include "opacity_masks.h"

namespace pt {

struct HitRecord { float t, u, v; uint gid; };      // gid == 0xFFFFFFFF: miss

constexpr int kTraversalStackSize = 32;

// Round-to-nearest IEEE operations that keep subnormals whatever -ftz / -use_fast_math says (inline PTX is not rewritten by those flags):
// the hit records have to be bit-identical to the oracle's in every build.
PT_DEVICE float xmul(float a, float b) { float r; asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
PT_DEVICE float xadd(float a, float b) { float r; asm("add.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
PT_DEVICE float xsub(float a, float b) { float r; asm("sub.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
PT_DEVICE float xdiv(float a, float b) { float r; asm("div.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
PT_DEVICE float xedge64(float a, float b, float c, float d)        // float(double(a) * double(b) - double(c) * double(d)), each step rounded to nearest
{
    float r;
    asm("{ .reg .f64 da, db, dc, dd, p0, p1;\n\t"
        "cvt.f64.f32 da, %1; cvt.f64.f32 db, %2; cvt.f64.f32 dc, %3; cvt.f64.f32 dd, %4;\n\t"
        "mul.rn.f64 p0, da, db; mul.rn.f64 p1, dc, dd; sub.rn.f64 p0, p0, p1;\n\t"
        "cvt.rn.f32.f64 %0, p0; }" : "=f"(r) : "f"(a), "f"(b), "f"(c), "f"(d));
    return r;
}

struct WatertightRay
{
    int kx, ky, kz; float Sx, Sy, Sz;
    PT_DEVICE void setup(float3 d)
    {
        float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
        kz = (ax >= ay) ? ((ax >= az) ? 0 : 2) : ((ay >= az) ? 1 : 2);
        kx = (kz + 1) % 3; ky = (kx + 1) % 3;
        float dk = (kz == 0) ? d.x : ((kz == 1) ? d.y : d.z);
        if (dk < 0.0f) { int t = kx; kx = ky; ky = t; }
        float dx = (kx == 0) ? d.x : ((kx == 1) ? d.y : d.z);
        float dy = (ky == 0) ? d.x : ((ky == 1) ? d.y : d.z);
        Sx = xdiv(dx, dk); Sy = xdiv(dy, dk); Sz = xdiv(1.0f, dk);
    }
};

PT_DEVICE float comp(float3 v, int k) { return (k == 0) ? v.x : ((k == 1) ? v.y : v.z); }

PT_DEVICE bool intersectTriangleWatertight(const WatertightRay& wr, float3 org, float3 v0, float3 v1, float3 v2, float tMin, float tMax,
                                           float& tOut, float& uOut, float& vOut)
{
    const float3 A = mk3(xsub(v0.x, org.x), xsub(v0.y, org.y), xsub(v0.z, org.z));
    const float3 B = mk3(xsub(v1.x, org.x), xsub(v1.y, org.y), xsub(v1.z, org.z));
    const float3 C = mk3(xsub(v2.x, org.x), xsub(v2.y, org.y), xsub(v2.z, org.z));
    const float Akz = comp(A, wr.kz), Bkz = comp(B, wr.kz), Ckz = comp(C, wr.kz);
    const float Ax = xsub(comp(A, wr.kx), xmul(wr.Sx, Akz)), Ay = xsub(comp(A, wr.ky), xmul(wr.Sy, Akz));
    const float Bx = xsub(comp(B, wr.kx), xmul(wr.Sx, Bkz)), By = xsub(comp(B, wr.ky), xmul(wr.Sy, Bkz));
    const float Cx = xsub(comp(C, wr.kx), xmul(wr.Sx, Ckz)), Cy = xsub(comp(C, wr.ky), xmul(wr.Sy, Ckz));
    float U = xsub(xmul(Cx, By), xmul(Cy, Bx));
    float V = xsub(xmul(Ax, Cy), xmul(Ay, Cx));
    float W = xsub(xmul(Bx, Ay), xmul(By, Ax));
    if (U == 0.0f || V == 0.0f || W == 0.0f)
    {
        U = xedge64(Cx, By, Cy, Bx);
        V = xedge64(Ax, Cy, Ay, Cx);
        W = xedge64(Bx, Ay, By, Ax);
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = xadd(xadd(U, V), W);
    if (det == 0.0f) return false;
    const float Az = xmul(wr.Sz, Akz), Bz = xmul(wr.Sz, Bkz), Cz = xmul(wr.Sz, Ckz);
    const float T = xadd(xadd(xmul(U, Az), xmul(V, Bz)), xmul(W, Cz));
    const float t = xdiv(T, det);
    if (!(t > tMin && t < tMax)) return false;
    tOut = t; uOut = xdiv(V, det); vOut = xdiv(W, det);
    return true;
}

// AlphaTestImpl (BridgeDonut:929-971): true when the candidate is opaque at (u,v).  The three texture coordinates come from the triangle's
// shading record (scene_device.cuh) instead of the index / vertex buffer chain.
PT_DEVICE bool alphaTestPasses(const SceneView& sc, const RtxptSubInstanceData& s, uint gid, float u, float v)
{
    const uint4* rec = sc.triShade + size_t(gid) * kTriShadeWords;
    const uint4 r3 = __ldg(rec + 3), r4 = __ldg(rec + 4);
    const float2 t0 = mk2(__uint_as_float(r3.x), __uint_as_float(r3.y)), t1 = mk2(__uint_as_float(r3.z), __uint_as_float(r3.w)), t2 = mk2(__uint_as_float(r4.x), __uint_as_float(r4.y));
    const float b0 = 1.0f - (u + v);
    const float2 uv = mk2(t0.x * b0 + t1.x * u + t2.x * v, t0.y * b0 + t1.y * u + t2.y * v);
    const float opacity = tex2DLod<float4>(sc.textures[s.FlagsAndAlphaInfo & 0xFFFF], uv.x, uv.y, 0.0f).w;
    return opacity >= float(s.FlagsAndAlphaInfo >> 24) / 255.0f;
}

// Candidate hit on an alpha-tested triangle: the opacity mask first (the OMM analogue, opacity_masks.h) - a known micro-triangle decides without the texture fetch - then
// AlphaTestImpl.  Kept out of line: alpha-tested candidates are rare, and inlined this body costs the traversal loop registers it does not have (64 at 4 CTAs per SM).
__device__ __noinline__ bool alphaCandidateIsOpaque(const SceneView& sc, uint sub, uint gid, uint maskSlot, float u, float v)
{
    if (maskSlot != om::kNoMask)
    {
        const uint m = om::microIndex(u, v);
        const uint state = (__ldg(reinterpret_cast<const uint*>(sc.opacityMasks + maskSlot) + (m >> 4)) >> ((m & 15u) * 2u)) & 3u;
        if (state == om::kTransparent) return false;
        if (state == om::kOpaque) return true;
    }
    return alphaTestPasses(sc, sc.subInstances[sub & kTriSubInstanceMask], gid, u, v);
}

struct TraversalCounters { uint nodeVisits, triTests; };

// byte j of a packed word -> 1 + b * 2^-15, built by placing the byte in mantissa bits 8..15 of 1.0f (one PRMT)
PT_DEVICE float byteToUnitFloat(uint w, int j) { return __uint_as_float(__byte_perm(w, 0x3F800000u, 0x7604u | (uint(j) << 4))); }
#ifndef PT_I2F_AXES
#define PT_I2F_AXES 2       // how many of the three axes convert their bytes with I2F (XU pipe) instead of PRMT (ALU pipe): 2 spreads the conversions over both pipes.
                            // H100 SXM (700 W), bench.py ms/frame: 1 axis 23.50, 2 axes 23.16-23.18, 3 axes 23.59
#endif
// the same permute with the selector as an immediate: `one` is 0x3F800000 held in a register the compiler cannot see through (otherwise ptxas folds it into the
// instruction's only immediate slot and spends a second instruction per byte on moving the selector into a register - 16 per node visit in the round-1 SASS)
PT_DEVICE float byteToUnitFloatImm(uint w, int j, uint one)
{
    uint r;
    switch (j)
    {
    case 0: asm("prmt.b32 %0, %1, %2, 0x7604;" : "=r"(r) : "r"(w), "r"(one)); break;
    case 1: asm("prmt.b32 %0, %1, %2, 0x7614;" : "=r"(r) : "r"(w), "r"(one)); break;
    case 2: asm("prmt.b32 %0, %1, %2, 0x7624;" : "=r"(r) : "r"(w), "r"(one)); break;
    default: asm("prmt.b32 %0, %1, %2, 0x7634;" : "=r"(r) : "r"(w), "r"(one)); break;
    }
    return __uint_as_float(r);
}
#ifndef PT_PRMT_IMM
#define PT_PRMT_IMM 0      // immediate PRMT selectors: the saved selector moves are re-spent on re-materialising the constant (H100 SXM, 700 W, bench.py: 23.27 ms/frame with, 23.16-23.18 without)
#endif
template <bool I2F> PT_DEVICE float byteToCoord(uint w, int j, uint one) { return I2F ? float((w >> (8 * j)) & 0xFFu) : (PT_PRMT_IMM ? byteToUnitFloatImm(w, j, one) : byteToUnitFloat(w, j)); }

// ---- warp-cooperative traversal ------------------------------------------------------------------------------------------------------
// Node steps are per-lane work (each lane walks its own ray through the CWBVH8).  Triangle tests are NOT: a leaf holds 1..3 triangles and
// only about a third of the lanes reach a leaf in any given step, so testing them lane-by-lane leaves the warp at ~8 % utilisation in that
// phase (ncu, round 1: 12 of 32 threads active per instruction overall).  Instead every lane appends its (ray lane, triangle) pairs to a
// ring buffer in shared memory that belongs to the warp, and the warp drains it 32 pairs at a time — any lane tests any ray's triangle,
// reading that ray from shared memory.  Hits are merged into the owner's record with a 64-bit shared-memory atomicMin on the key
// (bits(t) << 32 | gid), which is exactly the "smaller t, ties to the smaller global triangle id" rule, so the result does not depend on
// the order in which pairs are drained (and a stale pair that is tested against a lane's next ray is only a redundant, valid test).
#ifndef PT_PREFETCH_CHILDREN
#define PT_PREFETCH_CHILDREN 0
#endif
constexpr uint kTriQueueSize = 128;         // ring entries per warp (power of two)
constexpr uint kTriOwnerShift = 27;         // entry = owner lane << 27 | triangle index   (upload_scene rejects scenes with >= 2^27 triangles)

struct WarpScratch
{
    float ray[9][32];                       // per lane: org.xyz, Sx, Sy, Sz, kx|ky<<2|kz<<4 (bits), tMin, tMax
    unsigned long long bestKey[32];         // bits(t) << 32 | gid ; gid 0xFFFFFFFF = nothing accepted yet (t = tMax)
    float bestU[32], bestV[32];
    uint bestSub[32];
    uint queue[kTriQueueSize];
    uint tail, pad[3];                      // ring reservation cursor (the consumer cursor `head` is warp-uniform and lives in registers)
};
static_assert(sizeof(WarpScratch) == 2320, "WarpScratch layout");

// Resumable per-lane traversal state.  A persistent warp keeps one Traverser per lane; run() is called by all 32 lanes and advances every
// unfinished ray until fewer than `minActiveLanes` of them are left, so that the caller can fetch new rays for the idle lanes (dynamic
// fetch, Aila & Laine HPG 2009).  The traversal stack is a separate local array owned by the kernel so that the scalar state stays in
// registers; head/tail are the warp-uniform ring cursors.
template <bool ANY_HIT, bool COUNT>
struct Traverser
{
    float3 org;
    float idx, idy, idz, tMin, bestT;
    uint2 nodeGroup;
    uint octinv, lastTicket;
    int sp;
    bool done, waiting;

    PT_DEVICE void init(const SceneView& sc, WarpScratch& ws, float3 o, float3 d, float tmin, float tmax)
    {
        const uint lane = threadIdx.x & 31u;
        org = o; tMin = tmin; bestT = tmax;
        WatertightRay wr; wr.setup(d);
        ws.ray[0][lane] = o.x; ws.ray[1][lane] = o.y; ws.ray[2][lane] = o.z;
        ws.ray[3][lane] = wr.Sx; ws.ray[4][lane] = wr.Sy; ws.ray[5][lane] = wr.Sz;
        ws.ray[6][lane] = __uint_as_float(uint(wr.kx) | (uint(wr.ky) << 2) | (uint(wr.kz) << 4));
        ws.ray[7][lane] = tmin; ws.ray[8][lane] = tmax;
        ws.bestKey[lane] = ((unsigned long long)__float_as_uint(tmax) << 32) | 0xFFFFFFFFull;
        const float eps = 1.0e-20f;     // keeps s * id * 2^15 finite for every node scale the builder emits
        // reciprocal directions feed the conservative box test only: the 1-ulp approximation is inside its slack
        idx = __fdividef(1.0f, fabsf(d.x) > eps ? d.x : copysignf(eps, d.x));
        idy = __fdividef(1.0f, fabsf(d.y) > eps ? d.y : copysignf(eps, d.y));
        idz = __fdividef(1.0f, fabsf(d.z) > eps ? d.z : copysignf(eps, d.z));
        octinv = 7u - ((d.x < 0.0f ? 4u : 0u) | (d.y < 0.0f ? 2u : 0u) | (d.z < 0.0f ? 1u : 0u));
        sp = 0;
        nodeGroup = make_uint2(0u, 0x80000000u);        // virtual parent of the root: one internal child in slot 7^octinv
        waiting = false; lastTicket = 0;
        done = (sc.bvhTriCount == 0) || !(tmax > tmin);
    }

    PT_DEVICE static HitRecord result(const WarpScratch& ws, uint& subInstance)
    {
        const uint lane = threadIdx.x & 31u;
        const unsigned long long key = ws.bestKey[lane];
        HitRecord r; r.gid = uint(key); r.t = __uint_as_float(uint(key >> 32)); r.u = ws.bestU[lane]; r.v = ws.bestV[lane]; subInstance = ws.bestSub[lane];
        if (r.gid == 0xFFFFFFFFu) { r.t = -1.0f; r.u = 0.f; r.v = 0.f; subInstance = 0; }
        return r;
    }

    // drains `n` ring entries starting at `first`: lane L tests entries first+L, first+L+32, ...
    PT_DEVICE static void testEntries(const SceneView& sc, WarpScratch& ws, uint first, uint n, TraversalCounters* counters)
    {
        const uint lane = threadIdx.x & 31u;
        for (uint base = 0; base < n; base += 32u)
        {
            bool won = false; unsigned long long key = 0; float u = 0.f, v = 0.f; uint owner = 0, sub = 0;
            if (base + lane < n)
            {
                const uint ent = ws.queue[(first + base + lane) & (kTriQueueSize - 1u)];
                owner = ent >> kTriOwnerShift;
                const float4* tp = sc.bvhTris + size_t(ent & ((1u << kTriOwnerShift) - 1u)) * 3;
                const float4 a = __ldg(tp), b = __ldg(tp + 1), c = __ldg(tp + 2);
                if (COUNT) counters->triTests++;
                WatertightRay wr; const uint kp = __float_as_uint(ws.ray[6][owner]);
                wr.kx = int(kp & 3u); wr.ky = int((kp >> 2) & 3u); wr.kz = int(kp >> 4);
                wr.Sx = ws.ray[3][owner]; wr.Sy = ws.ray[4][owner]; wr.Sz = ws.ray[5][owner];
                float t;
                if (intersectTriangleWatertight(wr, mk3(ws.ray[0][owner], ws.ray[1][owner], ws.ray[2][owner]), mk3(a.x, a.y, a.z), mk3(b.x, b.y, b.z), mk3(c.x, c.y, c.z),
                                                ws.ray[7][owner], ws.ray[8][owner], t, u, v))
                {
                    key = ((unsigned long long)__float_as_uint(t) << 32) | __float_as_uint(a.w);
                    sub = __float_as_uint(b.w);
                    if (key < ws.bestKey[owner])
                    {
                        bool accept = true;
                        if (sub & (kTriFlagAlphaTested | kTriFlagExcludeFromNEE))
                        {   // non-opaque geometry (SampleCommon/AccelerationStructureUtil.h:88-89)
                            if (ANY_HIT && (sub & kTriFlagExcludeFromNEE)) accept = false;
                            else if ((sub & kTriFlagAlphaTested) && !alphaCandidateIsOpaque(sc, sub, __float_as_uint(a.w), __float_as_uint(c.w), u, v)) accept = false;
                        }
                        if (accept) { atomicMin(&ws.bestKey[owner], key); won = true; }
                    }
                }
            }
            __syncwarp();
            if (won && ws.bestKey[owner] == key) { ws.bestU[owner] = u; ws.bestV[owner] = v; ws.bestSub[owner] = sub & kTriSubInstanceMask; }
            __syncwarp();
        }
    }

    // All 32 lanes of the warp call this together.
    PT_DEVICE void run(const SceneView& sc, const uint4* __restrict__ nodes, const uint4* __restrict__ smemNodes, uint smemNodeCount, int minActiveLanes, int waitFlushLanes,
                       TraversalCounters* counters, uint2* __restrict__ stack, WarpScratch& ws, uint& head, uint& tail)
    {
        const uint lane = threadIdx.x & 31u;
        const uint octinv4 = octinv * 0x01010101u;
        const bool negx = !(octinv & 4u), negy = !(octinv & 2u), negz = !(octinv & 1u);
        uint one; asm volatile("mov.b32 %0, 0x3F800000;" : "=r"(one));        // see byteToUnitFloatImm
        while (true)
        {
            uint triBase = 0, triBits = 0;
            const bool traversing = !done && !waiting;
            if (traversing)
            {
                const uint hits = nodeGroup.y;
                const uint bitIndex = 31u - __clz(hits & 0xFF000000u);
                nodeGroup.y &= ~(1u << bitIndex);
                if (nodeGroup.y & 0xFF000000u) { if (sp < kTraversalStackSize) stack[sp++] = nodeGroup; }
                const uint slot = (bitIndex - 24u) ^ octinv;
                const uint rel = __popc(hits & ~(0xFFFFFFFFu << slot) & 0xFFu);
                const uint nodeIndex = nodeGroup.x + rel;
                uint4 n0, n1, n2, n3, n4;
                if (smemNodeCount == 0)
                {   // default: the whole BVH is read through L1 (read-only path); measured faster than giving L1 capacity away to a staged prefix
                    const uint4* np = nodes + size_t(nodeIndex) * 5;
                    n0 = __ldg(np); n1 = __ldg(np + 1); n2 = __ldg(np + 2); n3 = __ldg(np + 3); n4 = __ldg(np + 4);
                }
                else
                {
                    const uint4* np = (nodeIndex < smemNodeCount) ? (smemNodes + nodeIndex * 5) : (nodes + size_t(nodeIndex) * 5);
                    n0 = np[0]; n1 = np[1]; n2 = np[2]; n3 = np[3]; n4 = np[4];
                }
                if (COUNT) counters->nodeVisits++;

                const float px = __uint_as_float(n0.x), py = __uint_as_float(n0.y), pz = __uint_as_float(n0.z);
                // quantisation scale 2^(e-127) per axis, times 2^15 (bvh_builder.cpp keeps e + 15 < 255)
                const float sx15 = __uint_as_float(((n0.w & 0xFFu) + 15u) << 23), sy15 = __uint_as_float((((n0.w >> 8) & 0xFFu) + 15u) << 23), sz15 = __uint_as_float((((n0.w >> 16) & 0xFFu) + 15u) << 23);
                const uint imask = n0.w >> 24;
                nodeGroup.x = n1.x; triBase = n1.y;
                // Slab test on the quantised child boxes.  A quantised coordinate byte b is turned into the float m = 1 + b * 2^-15 with one
                // byte permute (ALU pipe) instead of an integer->float conversion (quarter-rate XU pipe, the top pipe of this kernel in the
                // round-1 ncu capture); then b * (s * id) + o == m * A + (o - A) with A = s * id * 2^15.  The box test only has to be
                // conservative (the triangle test decides): the relative slack eps and an absolute pad that covers the rounding of (o - A)
                // (<= 2^-22 (|A| + |o|), |o| <= |t| + 2^8 |s id|) are folded into the per-node constants, near planes pulled in, far pushed out.
                // PT_I2F_AXES of the three axes keep the integer->float conversion (XU pipe) so that the conversions are spread over two pipes:
                // for those, b * (s id) + o is evaluated directly (A = s id, no offset), with the same slack.
                const float Ax15 = sx15 * idx, Ay15 = sy15 * idy, Az15 = sz15 * idz;
                const float Ax = (PT_I2F_AXES > 0) ? Ax15 * (1.0f / 32768.0f) : Ax15, Ay = (PT_I2F_AXES > 1) ? Ay15 * (1.0f / 32768.0f) : Ay15, Az = (PT_I2F_AXES > 2) ? Az15 * (1.0f / 32768.0f) : Az15;
                const float ox = (px - org.x) * idx, oy = (py - org.y) * idy, oz = (pz - org.z) * idz;
                const float Ox = (PT_I2F_AXES > 0) ? ox : ox - Ax, Oy = (PT_I2F_AXES > 1) ? oy : oy - Ay, Oz = (PT_I2F_AXES > 2) ? oz : oz - Az;
                const float kLo = 1.0f - 6.0e-7f, kHi = 1.0f + 6.0e-7f, kPad = 4.8e-7f;
                const float Anx = Ax * kLo, Any = Ay * kLo, Anz = Az * kLo, Afx = Ax * kHi, Afy = Ay * kHi, Afz = Az * kHi;
                const float Onx = __fmaf_rn(Ox, kLo, -fabsf(Ax15) * kPad), Ony = __fmaf_rn(Oy, kLo, -fabsf(Ay15) * kPad), Onz = __fmaf_rn(Oz, kLo, -fabsf(Az15) * kPad);
                const float Ofx = __fmaf_rn(Ox, kHi, fabsf(Ax15) * kPad), Ofy = __fmaf_rn(Oy, kHi, fabsf(Ay15) * kPad), Ofz = __fmaf_rn(Oz, kHi, fabsf(Az15) * kPad);
                uint hitmask = 0;
                #pragma unroll
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
                    #pragma unroll
                    for (int j = 0; j < 4; j++)
                    {
                        const float t0x = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 0)>(nearx, j, one), Anx, Onx), t1x = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 0)>(farx, j, one), Afx, Ofx);
                        const float t0y = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 1)>(neary, j, one), Any, Ony), t1y = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 1)>(fary, j, one), Afy, Ofy);
                        const float t0z = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 2)>(nearz, j, one), Anz, Onz), t1z = __fmaf_rn(byteToCoord<(PT_I2F_AXES > 2)>(farz, j, one), Afz, Ofz);
                        const float cmin = fmaxf(fmaxf(t0x, t0y), fmaxf(t0z, tMin));
                        const float cmax = fminf(fminf(t1x, t1y), fminf(t1z, bestT));
                        if (cmin <= cmax)
                            hitmask |= ((childBits4 >> (8 * j)) & 0xFFu) << ((bitIndex4 >> (8 * j)) & 0xFFu);
                    }
                }
                nodeGroup.y = (hitmask & 0xFF000000u) | imask;
                triBits = hitmask & 0x00FFFFFFu;
                if (PT_PREFETCH_CHILDREN)
                {   // every hit inner child will be visited (popped groups are not re-tested): pull the ones that are not next into L1/L2 now
                    uint rest = nodeGroup.y & 0xFF000000u;
                    rest &= ~(0x80000000u >> __clz(rest));          // all but the child the next step descends into
                    while (rest)
                    {
                        const uint bi = 31u - __clz(rest); rest &= ~(1u << bi);
                        const uint sl = (bi - 24u) ^ octinv;
                        const uint4* cp = nodes + size_t(nodeGroup.x + __popc(imask & ~(0xFFFFFFFFu << sl))) * 5;
                        asm volatile("prefetch.global.L1 [%0];" ::"l"(cp));
                    }
                }
                if ((nodeGroup.y & 0xFF000000u) == 0)
                {
                    if (sp == 0) waiting = true; else nodeGroup = stack[--sp];
                }
            }

            // append this step's (lane, triangle) pairs to the warp's ring: every lane reserves its span with one shared-memory atomic
            // (order is irrelevant, see above).  Spans that would overrun the ring are given back: they are the tail of the reservation
            // order, so the valid entries stay a prefix; the ring is drained and those lanes try again.
            uint cnt = __popc(triBits);
            if (__any_sync(0xFFFFFFFFu, cnt != 0))
            {
                while (true)
                {
                    uint off = 0;
                    if (cnt) off = atomicAdd(&ws.tail, cnt);
                    __syncwarp();
                    const uint reserved = ws.tail, limit = head + kTriQueueSize;
                    const bool fits = cnt != 0 && int(off + cnt - limit) <= 0;
                    if (fits)
                    {
                        const uint tag = (lane << kTriOwnerShift) | triBase;
                        do
                        {
                            const uint k = __ffs(triBits) - 1u; triBits &= triBits - 1u;
                            ws.queue[off & (kTriQueueSize - 1u)] = tag + k;
                            off++;
                        } while (triBits != 0);
                        lastTicket = off; cnt = 0;
                    }
                    if (int(reserved - limit) <= 0) { tail = reserved; __syncwarp(); break; }
                    tail = head + __reduce_min_sync(0xFFFFFFFFu, cnt ? off - head : kTriQueueSize);
                    __syncwarp();
                    testEntries(sc, ws, head, tail - head, counters); head = tail;
                    if (lane == 0) ws.tail = tail;
                    __syncwarp();
                }
            }

            // drain: whole groups of 32 pairs as soon as they exist; a partial group only when lanes are starving for their results
            {
                const uint avail = tail - head;
                const uint nWait = __popc(__ballot_sync(0xFFFFFFFFu, waiting && !done));
                const uint nTrav = __popc(__ballot_sync(0xFFFFFFFFu, !waiting && !done));
                const bool partial = avail != 0 && (nTrav == 0 || nWait >= uint(waitFlushLanes));
                if (avail >= 32u || partial)
                {
                    const uint n = partial ? avail : (avail & ~31u);
                    testEntries(sc, ws, head, n, counters); head += n;
                    const unsigned long long key = ws.bestKey[lane];
                    bestT = __uint_as_float(uint(key >> 32));
                    if (ANY_HIT && uint(key) != 0xFFFFFFFFu) done = true;
                }
                if (waiting && int(head - lastTicket) >= 0) done = true;
            }
            if (int(__popc(__ballot_sync(0xFFFFFFFFu, !done))) < minActiveLanes) return;        // let the warp refill its idle lanes
        }
    }
};

} // namespace pt
