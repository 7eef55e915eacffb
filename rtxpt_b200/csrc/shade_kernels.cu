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

// warp-aggregated append to counter `cls` (0xFF = nothing to append); every lane of the warp must call this.  Returns the lane's position.
PT_DEVICE uint warpAppend(uint* counters, uint cls)
{
    const uint lane = threadIdx.x & 31u;
    const uint peers = __match_any_sync(0xFFFFFFFFu, cls);
    uint base = 0;
    if (cls != 0xFFu)
    {
        const uint leader = __ffs(peers) - 1u;
        if (lane == leader) base = atomicAdd(counters + cls, __popc(peers));
        base = __shfl_sync(peers, base, leader) + __popc(peers & ((1u << lane) - 1u));
    }
    return base;
}

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
// MULTI (NEEFullSamples > 1): shadeHit appends the vertex's shadow records and NEE block itself, one record per valid light sample
template <int MINB, bool EXPORT_GUIDES, bool ANALYTIC_LIGHTS, bool NEEAT = false, bool MULTI = false>
__global__ void __launch_bounds__(128, MINB) k_shade(const __grid_constant__ LaunchParams p)
{
    uint* ctr = p.wf.counters + p.iteration * kCountersPerIter;
    uint* ctrNext = ctr + kCountersPerIter;
    const uint warpsPerBlock = blockDim.x >> 5, lane = threadIdx.x & 31u;
    const uint warpGlobal = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5), warpStride = gridDim.x * warpsPerBlock;
    for (int cls = 0; cls < kNumShadeClasses; cls++)
    {
        const uint count = ctr[kCtrShadeCount + cls];
        const uint* __restrict__ queue = p.wf.shadeQueue + size_t(cls) * p.wf.capacity;
        for (uint base = warpGlobal * 32u; base < count; base += warpStride * 32u)
        {
            const uint i = base + lane;
            uint rayCls = 0xFFu, shadowCls = 0xFFu, h = 0;
            PathRegs path;
            HitOutputs out; out.continuePath = false; out.emitShadow = false;
            if (i < count)
            {
                const uint r = queue[i];
                h = path.loadRay(p.stateIn, r, p.radiance);
                if constexpr (NEEAT) out.naRecord = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
                if (cls == 0) shadeMiss<EXPORT_GUIDES, kModeReference, NEEAT>(p, path);
                else shadeHit<EXPORT_GUIDES, ANALYTIC_LIGHTS, kModeReference, NEEAT, MULTI>(p, path, h, p.wf.hits[r], out);
                path.storeRadiance(p.radiance, h);
                if (out.continuePath) rayCls = 0;
                if (out.emitShadow) shadowCls = 0;
            }
            // a continuing path becomes a ray of the next iteration: appended to the other state set, so a warp's paths land in consecutive entries
            const uint next = warpAppend(ctrNext + kCtrRayCount, rayCls);
            if (rayCls == 0) path.storeRay(p.stateOut, next, h);
            // shadow records: warp-aggregated, long rays from the front of the three arrays, the rest from the back (appendShadowRecord)
            if constexpr (!MULTI)
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
    if (min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1)
    {   // several light samples per vertex: analytic lights compiled in, gated by the light type at run time
        if (p.exportGuides) k_shade<3, true, true, false, true><<<g.smCount * 3, 128, 0, s>>>(p); else k_shade<3, false, true, false, true><<<g.smCount * 3, 128, 0, s>>>(p);
        return;
    }
    if (p.exportGuides) { k_shade<4, true, true><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (p.scene.analyticLightCount != 0) { k_shade<4, false, true><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (g.shadeBlocksPerSM >= 5) k_shade<5, false, false><<<grid, 128, 0, s>>>(p);
    else if (g.shadeBlocksPerSM == 4) k_shade<4, false, false><<<grid, 128, 0, s>>>(p);
    else k_shade<3, false, false><<<grid, 128, 0, s>>>(p);
}
void launchDebugBsdf(const float* in, uint32_t count, float* out, cudaStream_t s) { k_debug_bsdf<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }
void launchDebugRng(const uint32_t* in, uint32_t count, uint32_t* out, cudaStream_t s) { k_debug_rng<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }


} // namespace pt
