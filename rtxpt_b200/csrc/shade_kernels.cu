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
// AMIS: approximate light-vs-BSDF MIS (RtxptPathTracerConstants::useApproximateMIS = 1); a template argument, as RTXPT compiles it in
// STF: stochastic texture filtering of the material fetches (rtxpt_b200_set_texture_filtering); its kernels carry analytic lights, gated by the light type at run time
// DEBUG_VIEW: a first-hit debug view is set (rtxpt_b200_set_debug_view); its kernels carry analytic lights, gated by the light type at run time
template <int MINB, bool EXPORT_GUIDES, bool ANALYTIC_LIGHTS, bool NEEAT = false, bool MULTI = false, bool AMIS = false, bool STF = false, bool DEBUG_VIEW = false>
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
                if (cls == 0) shadeMiss<EXPORT_GUIDES, kModeReference, NEEAT, AMIS>(p, path);
                else shadeHit<EXPORT_GUIDES, ANALYTIC_LIGHTS, kModeReference, NEEAT, MULTI, AMIS, STF, DEBUG_VIEW>(p, path, h, p.wf.hits[r], out);
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

// first-hit debug view: the kernel the launch would run otherwise, with the view drawn at vertex 1; one instantiation per guide / sample-count / STF choice, analytic lights
// gated at run time, at the CTA count of the kernel it stands in for
template <int MINB, bool EXPORT_GUIDES, bool NEEAT, bool MULTI, bool AMIS, bool STF>
static void launchShadeDebugView(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_shade<MINB, EXPORT_GUIDES, true, NEEAT, MULTI, AMIS, STF, true><<<g.smCount * MINB, 128, 0, s>>>(p); }
template <bool AMIS, bool STF>
static void launchShadeDebugViewMis(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    if (min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1) { if (p.exportGuides) launchShadeDebugView<3, true, false, true, AMIS, STF>(p, g, s); else launchShadeDebugView<3, false, false, true, AMIS, STF>(p, g, s); }
    else { if (p.exportGuides) launchShadeDebugView<4, true, false, false, AMIS, STF>(p, g, s); else launchShadeDebugView<4, false, false, false, AMIS, STF>(p, g, s); }
}
static bool firstHitDebugView(const LaunchParams& p) { return p.dbg.viz && isFirstHitView(p.dbg.view); }

// reference mode with NEE-AT feedback: one instantiation per MIS kind (guides on: the feedback passes reproject with them; analytic lights compiled in, gated by the light type at run time)
void launchShadeNeeat(const LaunchParams& p, const GridConfig& g, cudaStream_t s)       // 3 CTAs per SM: 155 registers, no spills
{
    if (firstHitDebugView(p))
    {
        if (p.stf.pointTextures) { if (p.c.useApproximateMIS) launchShadeDebugView<3, true, true, false, true, true>(p, g, s); else launchShadeDebugView<3, true, true, false, false, true>(p, g, s); }
        else { if (p.c.useApproximateMIS) launchShadeDebugView<3, true, true, false, true, false>(p, g, s); else launchShadeDebugView<3, true, true, false, false, false>(p, g, s); }
        return;
    }
    if (p.stf.pointTextures)
    {
        if (p.c.useApproximateMIS) k_shade<3, true, true, true, false, true, true><<<g.smCount * 3, 128, 0, s>>>(p); else k_shade<3, true, true, true, false, false, true><<<g.smCount * 3, 128, 0, s>>>(p);
        return;
    }
    if (p.c.useApproximateMIS) k_shade<3, true, true, true, false, true><<<g.smCount * 3, 128, 0, s>>>(p); else k_shade<3, true, true, true><<<g.smCount * 3, 128, 0, s>>>(p);
}
// the same choice of kernel for either MIS kind: the approximate kernels are the full-MIS ones with AMIS set
template <bool AMIS>
static void launchShadeMis(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    const int grid = g.smCount * g.shadeBlocksPerSM;
    if (firstHitDebugView(p)) { if (p.stf.pointTextures) launchShadeDebugViewMis<AMIS, true>(p, g, s); else launchShadeDebugViewMis<AMIS, false>(p, g, s); return; }
    if (p.stf.pointTextures)
    {   // stochastic texture filtering: one kernel per guide / sample-count choice.  4 CTAs per SM although the single-sample kernels spill 12-24 bytes there: measured on an H100,
        // k_shade on the bench workload is 7.37 ms at 4 CTAs and 7.76 ms at 3 without spills.  Like the guide and analytic-light kernels, they do not follow RTXPT_SHADE_CTAS
        const bool multi = min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1;
        if (multi) { if (p.exportGuides) k_shade<3, true, true, false, true, AMIS, true><<<g.smCount * 3, 128, 0, s>>>(p); else k_shade<3, false, true, false, true, AMIS, true><<<g.smCount * 3, 128, 0, s>>>(p); }
        else { if (p.exportGuides) k_shade<4, true, true, false, false, AMIS, true><<<g.smCount * 4, 128, 0, s>>>(p); else k_shade<4, false, true, false, false, AMIS, true><<<g.smCount * 4, 128, 0, s>>>(p); }
        return;
    }
    // guide export and analytic (sphere) lights are separate instantiations: the default kernel carries neither
    if (min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1)
    {   // several light samples per vertex: analytic lights compiled in, gated by the light type at run time
        if (p.exportGuides) k_shade<3, true, true, false, true, AMIS><<<g.smCount * 3, 128, 0, s>>>(p); else k_shade<3, false, true, false, true, AMIS><<<g.smCount * 3, 128, 0, s>>>(p);
        return;
    }
    if (p.exportGuides) { k_shade<4, true, true, false, false, AMIS><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (p.scene.analyticLightCount != 0) { k_shade<4, false, true, false, false, AMIS><<<g.smCount * 4, 128, 0, s>>>(p); return; }
    if (g.shadeBlocksPerSM >= 5) k_shade<5, false, false, false, false, AMIS><<<grid, 128, 0, s>>>(p);
    else if (g.shadeBlocksPerSM == 4) k_shade<4, false, false, false, false, AMIS><<<grid, 128, 0, s>>>(p);
    else k_shade<3, false, false, false, false, AMIS><<<grid, 128, 0, s>>>(p);
}
void launchShade(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    if (p.c.useApproximateMIS) launchShadeMis<true>(p, g, s); else launchShadeMis<false>(p, g, s);
}
void launchDebugBsdf(const float* in, uint32_t count, float* out, cudaStream_t s) { k_debug_bsdf<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }
void launchDebugRng(const uint32_t* in, uint32_t count, uint32_t* out, cudaStream_t s) { k_debug_rng<<<(count + 127) / 128, 128, 0, s>>>(in, count, out); }


} // namespace pt
