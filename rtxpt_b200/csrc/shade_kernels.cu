// shade_kernels.cu — the shading half of the wavefront (see kernels.cu for the sequence): k_shade runs the ClosestHit / miss shader bodies of
// shade.cuh over the per-class queues written by k_trace_closest.  It is its own translation unit because the default build compiles it with
// -use_fast_math (approximate division, reciprocal, sqrt, sin/cos/exp2/log2 — the arithmetic a GPU shader compiler gives the reference's
// HLSL), while everything that produces hit records, camera rays and queue indices stays in kernels.cu under exact flags.  The strict build
// compiles both units with IEEE arithmetic.
#if !RTXPT_STRICT_FP
#define PT_FAST_MATH 1
#endif
#define PT_SOBOL_TABLES 1
#include "shade.cuh"
#include "kernels.h"

namespace pt {

// warp-aggregated append of `value` to queue region `cls` (0xFF = nothing to append); every lane of the warp must call this
PT_DEVICE void warpAppend(uint* queueBase, uint regionStride, uint* counters, uint cls, uint value)
{
    const uint lane = threadIdx.x & 31u;
    const uint peers = __match_any_sync(0xFFFFFFFFu, cls);
    if (cls != 0xFFu)
    {
        const uint leader = __ffs(peers) - 1u;
        uint base = 0;
        if (lane == leader) base = atomicAdd(counters + cls, __popc(peers));
        base = __shfl_sync(peers, base, leader);
        queueBase[size_t(cls) * regionStride + base + __popc(peers & ((1u << lane) - 1u))] = value;
    }
}

// next-item prefetch in k_shade: 0 off, 1 into L2, 2 into L1
#ifndef PT_SHADE_PREFETCH
#define PT_SHADE_PREFETCH 0
#endif
#if PT_SHADE_PREFETCH == 2
#define PT_PREFETCH(ptr) asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr))
#else
#define PT_PREFETCH(ptr) asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr))
#endif

__global__ void k_init_sobol_tables()
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < 4u * 4u * 256u; i += gridDim.x * blockDim.x)
    {
        const uint dim = i >> 10, byte = (i >> 8) & 3u, v = i & 0xFFu;
        gSobolByte[dim][byte][v] = sobolDimBitwise(v << (8u * byte), dim + 1u);
    }
}
void launchInitTables(cudaStream_t s) { k_init_sobol_tables<<<16, 256, 0, s>>>(); }

// ---- shade --------------------------------------------------------------------------------------------------------------------------------
template <int MINB, bool EXPORT_GUIDES, bool ANALYTIC_LIGHTS, bool NEEAT = false>
__global__ void __launch_bounds__(128, MINB) k_shade(const __grid_constant__ LaunchParams p)
{
    uint* ctr = p.wf.counters + p.iteration * kCountersPerIter;
    uint* ctrNext = ctr + kCountersPerIter;
    uint* nextQueue = p.wf.rayQueue[(p.iteration + 1) & 1];
    const uint warpsPerBlock = blockDim.x >> 5, lane = threadIdx.x & 31u;
    const uint warpGlobal = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5), warpStride = gridDim.x * warpsPerBlock;
    for (int cls = 0; cls < kNumShadeClasses; cls++)
    {
        const uint count = ctr[kCtrShadeCount + cls];
        const uint* __restrict__ queue = p.wf.shadeQueue + size_t(cls) * p.wf.capacity;
#if PT_SHADE_PREFETCH
        // Software pipeline over the queue (the kernel is latency-bound: 4 warps per scheduler, a chain of dependent gathers per path): while
        // item k is shaded, the state words and the hit of item k+1 are pulled towards the SM, and once its hit has arrived, its 96-byte shade record.
        uint slotNext = (warpGlobal * 32u + lane < count) ? queue[warpGlobal * 32u + lane] : 0xFFFFFFFFu;
#endif
        for (uint base = warpGlobal * 32u; base < count; base += warpStride * 32u)
        {
            const uint i = base + lane;
            uint rayCls = 0xFFu, shadowCls = 0xFFu, rayEntry = 0, slot = 0;
            HitOutputs out; out.continuePath = false; out.emitShadow = false;
#if PT_SHADE_PREFETCH
            const uint slotNow = slotNext;
            { const uint ni = i + warpStride * 32u; slotNext = ni < count ? queue[ni] : 0xFFFFFFFFu; }          // consumed after this item: the load has a whole item to land
#endif
            if (i < count)
            {
#if PT_SHADE_PREFETCH
                slot = slotNow;
#else
                slot = queue[i];
#endif
                PathRegs path; path.load(p.wf, slot, true);
                if constexpr (NEEAT) out.naRecord = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
#if PT_SHADE_PREFETCH
                const float4 hitNow = cls != 0 ? p.wf.hits[slot] : make_float4(0.f, 0.f, 0.f, 0.f);
                if (slotNext != 0xFFFFFFFFu)
                {   // next item's state and hit (its slot index was loaded an item ago)
                    PT_PREFETCH(p.wf.s0 + slotNext); PT_PREFETCH(p.wf.s1 + slotNext); PT_PREFETCH(p.wf.s2 + slotNext); PT_PREFETCH(p.wf.s3 + slotNext); PT_PREFETCH(p.wf.s4 + slotNext);
                    if (cls != 0) PT_PREFETCH(p.wf.hits + slotNext);
                }
                if (cls == 0) shadeMiss<EXPORT_GUIDES, kModeReference, NEEAT>(p, path);
                else shadeHit<EXPORT_GUIDES, ANALYTIC_LIGHTS, kModeReference, NEEAT>(p, path, slot, hitNow, out);
                if (cls != 0 && slotNext != 0xFFFFFFFFu)
                {   // by now the next hit is close: its triangle's shade record (96 B = one or two 128-byte lines)
                    const uint gidNext = __float_as_uint(p.wf.hits[slotNext].w);
                    const uint4* rec = p.scene.triShade + size_t(gidNext) * kTriShadeWords;
                    PT_PREFETCH(rec); PT_PREFETCH(rec + 5);
                }
#else
                if (cls == 0) shadeMiss<EXPORT_GUIDES, kModeReference, NEEAT>(p, path);
                else shadeHit<EXPORT_GUIDES, ANALYTIC_LIGHTS, kModeReference, NEEAT>(p, path, slot, p.wf.hits[slot], out);
#endif
                if (cls != 0 && out.continuePath) path.store(p.wf, slot); else path.storeRadianceOnly(p.wf, slot);
                if (out.continuePath) { rayCls = 0; rayEntry = slot | (path.hasFlag(kPFTerminateAtNextBounce) ? 0x80000000u : 0u); }
                if (out.emitShadow) shadowCls = 0;
            }
            warpAppend(nextQueue, 0, ctrNext + kCtrRayCount, rayCls, rayEntry);
            // shadow records: warp-aggregated, long rays from the front of the three arrays, the rest from the back (appendShadowRecord)
            {
                const uint b = appendShadowRecord(p, ctr, shadowCls == 0, out.shadow.originTMax.w);
                if (shadowCls == 0)
                {
                    p.wf.shadowOriginTMax[b] = out.shadow.originTMax; p.wf.shadowDirPath[b] = out.shadow.dirPath; p.wf.shadowRadiance[b] = out.shadow.radiance;
                    if constexpr (NEEAT) p.naShadowFeedback[b] = out.naRecord;
                }
            }
        }
    }
}

// ---- debug: BSDF / RNG on the device (parity tests) -------------------------------------------------------------------------------------------
__global__ void k_debug_bsdf(const float* __restrict__ in, uint count, float* __restrict__ out)
{
    const uint i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const float* r = in + size_t(i) * 36; float* o = out + size_t(i) * 16;
    BsdfParams d;
    d.diffuse = mk3(r[18], r[19], r[20]); d.roughness = r[21]; d.specular = mk3(r[22], r[23], r[24]); d.metallic = r[25];
    d.transmission = mk3(r[26], r[27], r[28]); d.diffuseTransmission = r[29]; d.specularTransmission = r[30]; d.eta = r[31];
    BsdfSetup b; b.init(mk3(r[6], r[7], r[8]), mk3(r[9], r[10], r[11]), mk3(r[3], r[4], r[5]), mk3(r[0], r[1], r[2]), r[32] != 0.0f, d);
    const float3 wo = mk3(r[12], r[13], r[14]);
    const float4 e = b.eval(wo);
    o[0] = e.x; o[1] = e.y; o[2] = e.z; o[3] = e.w; o[4] = b.pdf(wo);
    BsdfSample s; const bool valid = b.sample(r[15], r[16], r[17], s);
    o[5] = valid ? 1.0f : 0.0f; o[6] = s.wo.x; o[7] = s.wo.y; o[8] = s.wo.z; o[9] = s.pdf; o[10] = s.weight.x; o[11] = s.weight.y; o[12] = s.weight.z;
    o[13] = float(s.lobe); o[14] = s.lobeP; o[15] = float(bsdfLobes(d));
}
__global__ void k_debug_rng(const uint* __restrict__ in, uint count, uint* __restrict__ out)
{
    const uint i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint baseHash = vertexBaseHash((in[i * 4] << 16) | in[i * 4 + 1], in[i * 4 + 2]);
    UniformSeq u = UniformSeq::make(baseHash, in[i * 4 + 3], 0u);
    for (int k = 0; k < 4; k++) out[i * 8 + k] = u.nextBits();
    for (uint k = 0; k < 4; k++) out[i * 8 + 4 + k] = __float_as_uint(hashToFloat(ldSampleBits(baseHash, in[i * 4 + 3], 1u, k)));
}

// reference mode with NEE-AT feedback: one instantiation (guides on: the feedback passes reproject with them; analytic lights compiled in, gated by the light type at run time)
void launchShadeNeeat(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_shade<3, true, true, true><<<g.smCount * 3, 128, 0, s>>>(p); }      // 3 CTAs per SM: 155 registers, no spills
void launchShade(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    const int grid = g.smCount * g.shadeBlocksPerSM;
    // guide export and analytic (sphere) lights are separate instantiations: the default kernel carries neither
    if (p.exportGuides) { k_shade<4, true, true><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (p.scene.analyticLightCount != 0) { k_shade<4, false, true><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (g.shadeBlocksPerSM >= 5) k_shade<5, false, false><<<grid, 128, 0, s>>>(p);
    else if (g.shadeBlocksPerSM == 4) k_shade<4, false, false><<<grid, 128, 0, s>>>(p);
    else k_shade<3, false, false><<<grid, 128, 0, s>>>(p);
}
void launchDebugBsdf(const float* in, uint32_t count, float* out, cudaStream_t s) { k_debug_bsdf<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }
void launchDebugRng(const uint32_t* in, uint32_t count, uint32_t* out, cudaStream_t s) { k_debug_rng<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }


} // namespace pt
