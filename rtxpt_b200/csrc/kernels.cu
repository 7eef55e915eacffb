// kernels.cu — the wavefront: generate -> [ trace closest -> shade (per material class) -> trace shadow ]* -> commit + accumulate.
//
// One launch of this sequence replaces one DispatchRays of the reference's megakernel (Rtxpt/Sample.cpp:2503-2517,
// Rtxpt/Shaders/PathTracerSample.hlsl:201-256), for `subSampleCount` sub-samples at once.
//   k_generate          EmptyPathInitialize + computeCameraRay (PathTracer.hlsli:47-91, BridgeDonut:543-564, PathTracerHelpers.hlsli:126-153)
//   k_trace_closest     Bridge::traceScatterRay (BridgeDonut:1029-1055) + the SER sort key: paths are binned by
//                       {miss, terminating hit, material class} (PathTracerSample.hlsl:136-148, MaterialsBaker.cpp:1267-1271)
//   k_shade             ClosestHit / miss shader bodies (shade.cuh; lives in shade_kernels.cu, which is compiled with fast-math flags)
//   k_trace_shadow      Bridge::traceVisibilityRay (BridgeDonut:993-1027) + the NEE radiance accumulation
//   k_commit_accumulate CommitPixel (PathTracer.hlsli:165-175) + AccumulationPass (ProcessingPasses/AccumulationPass.hlsl:36-66)
// All kernels are persistent (grid = SM count x resident CTAs) and read their work counts from device memory, so a whole frame is
// enqueued without a host round trip.  The top of the BVH (breadth-first prefix) is staged into shared memory with one TMA bulk copy
// per CTA (cp.async.bulk + mbarrier).
#include "device_math.cuh"
#include "traverse.cuh"
#include "kernels.h"

namespace pt {

// ---- TMA bulk copy global -> shared --------------------------------------------------------------------------------------------------
PT_DEVICE void stageNodesToShared(uint4* smemDst, const uint4* __restrict__ src, uint nodeCount, uint64_t* mbar)
{
    const uint bytes = nodeCount * 80u;
    const uint mbarAddr = (uint)__cvta_generic_to_shared(mbar);
    if (threadIdx.x == 0)
    {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbarAddr));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (bytes == 0) return;
    if (threadIdx.x == 0)
    {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbarAddr), "r"(bytes) : "memory");
        const uint chunk = 32768u;
        for (uint off = 0; off < bytes; off += chunk)
        {
            const uint n = min(chunk, bytes - off);
            const uint dst = (uint)__cvta_generic_to_shared(reinterpret_cast<char*>(smemDst) + off);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(reinterpret_cast<const char*>(src) + off), "r"(n), "r"(mbarAddr) : "memory");
        }
    }
    uint done = 0;
    while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(mbarAddr) : "memory");
}

// ---- generate --------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_generate(const __grid_constant__ LaunchParams p)
{
    const uint total = p.wf.pixelCount * p.subSampleCount;
    if (blockIdx.x == 0 && threadIdx.x == 0) p.wf.counters[kCtrRayCount] = total;     // iteration 0 traces every path's camera ray
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < total; slot += gridDim.x * blockDim.x)
    {
        const uint sub = slot / p.wf.pixelCount, pix = slot - sub * p.wf.pixelCount;
        const uint id = p.wf.pixelOfSlot[pix];
        const uint px = id >> 16, py = id & 0xFFFF;
        const uint sampleIndex = p.firstSampleIndex + sub;
        PathRegs path;
        path.id = id; path.sceneLength = 0.f; path.sampleIndex = sampleIndex;
        path.flagsAndVertexIndex = 0; path.packedCounters = 0; path.interior0 = path.interior1 = 0;
        path.setThp(mk3(1.f)); path.setL(make_float4(0.f, 0.f, 0.f, 0.f));
        path.setFlag(kPFActive, true); path.setFlag(kPFDeltaOnlyPath, true);
        path.setCone(0.f, p.c.camera.PixelConeSpreadAngle);
        path.setFireflyK_BsdfPdf(1.0f, 0.0f);
        path.setMisInfo_RuRu(0u, 1.0f);
        if (hasFinishedSurfaceBounces(p.c, 1, 0)) path.setFlag(kPFTerminateAtNextBounce, true);
        float3 origin, dir; computeCameraRay(p.c, id, sampleIndex, origin, dir);
        if (p.exportGuides && sub + 1 == p.subSampleCount) p.depth[size_t(py) * p.c.imageWidth + px] = 0.0f;       // Bridge::ExportSurfaceInit
        path.origin = origin; path.dir = dir;
        path.storeRay(p.stateIn, slot, slot);          // iteration 0: ray index == home index
        path.storeRadiance(p.radiance, slot);
    }
}

// ---- traversal loop -----------------------------------------------------------------------------------------------------------------------
// shared memory of the traversal kernels: [mbarrier 16 B][WarpScratch x 8 warps][staged BVH nodes]
#ifndef PT_TRACE_THREADS
#define PT_TRACE_THREADS 256     // threads per traversal CTA; the resident-CTA count scales so that warps per SM stay the same
#endif
constexpr uint kTraceThreads = PT_TRACE_THREADS, kTraceCtaScale = 256 / PT_TRACE_THREADS;
constexpr uint kTraceWarps = kTraceThreads / 32;
constexpr uint kTraceScratchBytes = 16 + kTraceWarps * sizeof(WarpScratch);

// Persistent warps with dynamic ray fetch, shared by every traversal kernel: a lane whose ray has finished retires it and pulls the next
// ray index from `fetchCursor` (one atomic per warp); lanes still traversing resume where they stopped.  Keeps SIMT lanes busy although
// ray lengths differ by an order of magnitude.  Rays 0 .. count-1 are traced; the callers differ only in the two inlined callbacks:
//   fetchRay(i, o, d, tMin, tMax)  loads ray i and keeps what the caller needs when the ray retires
//   retireRay(retireMask, ws)      called by every lane whose ray has finished, with its result in ws (Traverser::result); with RETIRE_MASK
//                                  retireMask is the ballot of those lanes, for warp-collective work among them (0 otherwise: no vote is taken)
// TMIN_ZERO: fetchRay gives every ray tMin == 0, which lets the node step compare distances as integers (traverse.cuh: nodeHitMask).
// Returns this thread's traversal counters (zero unless COUNT).
template <bool ANY_HIT, bool COUNT, bool RETIRE_MASK, bool TMIN_ZERO, typename FetchRay, typename RetireRay>
PT_DEVICE TraversalCounters traceLoop(const LaunchParams& p, uint* fetchCursor, uint count, FetchRay&& fetchRay, RetireRay&& retireRay)
{
    extern __shared__ __align__(16) unsigned char smemRaw[];
    uint64_t* mbar = reinterpret_cast<uint64_t*>(smemRaw);
    WarpScratch& ws = reinterpret_cast<WarpScratch*>(smemRaw + 16)[threadIdx.x >> 5];
    uint4* smemNodes = reinterpret_cast<uint4*>(smemRaw + kTraceScratchBytes);
    stageNodesToShared(smemNodes, p.scene.bvhNodes, p.smemNodeCount, mbar);

    TraversalCounters tc; tc.nodeVisits = 0; tc.triTests = 0;
    const uint lane = threadIdx.x & 31u, laneLt = (1u << lane) - 1u;
    Traverser<ANY_HIT, COUNT, TMIN_ZERO> tv; tv.done = true; tv.waiting = false;
    uint2 stack[kTraversalStackSize];
    uint head = 0, tail = 0;
    if (lane == 0) ws.tail = 0;
    __syncwarp();
    bool hasRay = false, exhausted = false;
    while (true)
    {
        const bool retire = tv.done && hasRay;
        const uint retireMask = RETIRE_MASK ? __ballot_sync(0xFFFFFFFFu, retire) : 0u;
        if (retire)
        {
            retireRay(retireMask, ws);
            hasRay = false;
        }
        // fetch the next ray for every idle lane with one atomic per warp
        const bool fetch = tv.done && !exhausted;
        const uint fetchMask = __ballot_sync(0xFFFFFFFFu, fetch);
        if (fetchMask)
        {
            const uint leader = __ffs(fetchMask) - 1u;
            uint base = 0;
            if (lane == leader) base = atomicAdd(fetchCursor, __popc(fetchMask));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
            if (fetch)
            {
                const uint i = base + __popc(fetchMask & laneLt);
                if (i >= count) exhausted = true;
                else
                {
                    float3 o, d; float tMin, tMax;
                    fetchRay(i, o, d, tMin, tMax);
                    tv.init(p.scene, ws, o, d, tMin, tMax);
                    hasRay = true;
                }
            }
        }
        __syncwarp();
        if (__all_sync(0xFFFFFFFFu, tv.done && !hasRay)) break;
        const bool drained = __any_sync(0xFFFFFFFFu, exhausted);
        tv.run(p.scene, p.scene.bvhNodes, smemNodes, p.smemNodeCount, drained ? 1 : p.refillThreshold, p.waitFlushLanes, &tc, stack, ws, head, tail);
    }
    return tc;
}

// ---- closest hit ------------------------------------------------------------------------------------------------------------------------
// A retiring lane writes its hit and bins the path into its shade queue.
// RAY_ORDER (reference mode): ray i is entry i of p.stateIn and writes hits[i]; otherwise (realtime) the ray queue names the path slot
template <bool COUNT, int MINB, bool RAY_ORDER>
__global__ void __launch_bounds__(kTraceThreads, MINB * kTraceCtaScale) k_trace_closest(const __grid_constant__ LaunchParams p)
{
    uint* ctr = p.wf.counters + p.iteration * kCountersPerIter;
    const uint count = ctr[kCtrRayCount];
    if (count == 0) return;                 // wavefront already drained (uniform across the grid)
    const uint* __restrict__ queue = p.wf.rayQueue[p.iteration & 1];
    uint entry = 0;
    auto fetchRay = [&](uint i, float3& o, float3& d, float& tMin, float& tMax)
    {
        uint4 a, b;
        if constexpr (RAY_ORDER)
        {   // the sign bit of s1.w is the path's kPFTerminateAtNextBounce (wavefront.cuh)
            a = ldState(p.stateIn.s0 + i); b = ldState(p.stateIn.s1 + i);
            entry = i | (b.w & 0x80000000u);
        }
        else
        {
            entry = queue[i];
            const uint slot = entry & 0x7FFFFFFFu;
            a = ldState(p.wf.s0 + slot); b = ldState(p.wf.s1 + slot);
        }
        o = mk3(__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z)); d = mk3(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z));
        tMin = 0.0f; tMax = kMaxRayTravel;
    };
    auto retireRay = [&](uint retireMask, const WarpScratch& ws)
    {   // hit record + SER-style binning by {miss, terminating hit, material class}
        const uint lane = threadIdx.x & 31u, laneLt = (1u << lane) - 1u;
        const uint slot = entry & 0x7FFFFFFFu;
        uint subInstance; const HitRecord h = Traverser<false, COUNT, true>::result(ws, subInstance);
        p.wf.hits[slot] = make_float4(h.t, h.u, h.v, __uint_as_float(h.gid));
        uint cls;
        if (h.gid == 0xFFFFFFFFu) cls = 0;
        else if (entry & 0x80000000u) cls = 1;
        else cls = (p.flags & RTXPT_CFG_NO_MATERIAL_SORT) ? 2u : 2u + p.scene.subInstanceClass[subInstance];
        const uint peers = __match_any_sync(retireMask, cls);
        const uint leader = __ffs(peers) - 1u;
        uint base = 0;
        if (lane == leader) base = atomicAdd(ctr + kCtrShadeCount + cls, __popc(peers));
        base = __shfl_sync(peers, base, leader);
        p.wf.shadeQueue[size_t(cls) * p.wf.capacity + base + __popc(peers & laneLt)] = slot;
    };
    const TraversalCounters tc = traceLoop<false, COUNT, true, true>(p, ctr + kCtrFetchClosest, count, fetchRay, retireRay);
    if (COUNT) { atomicAdd(ctr + kCtrNodeVisits, tc.nodeVisits); atomicAdd(ctr + kCtrTriTests, tc.triTests); }
}

// ---- shadow rays ----------------------------------------------------------------------------------------------------------------------------
// REALTIME (FILL pass of realtime mode): the radiance is attenuated by 1 / sub-sample count and comes with a specular average chosen by the shade
// kernel (sign bits of the record's first word, shade.cuh) - AccumulatePathRadiance of PATH_TRACER_MODE_FILL_STABLE_PLANES (PathTracer.hlsli:145-159)
// MULTI (NEEFullSamples > 1): a record is one light sample of a vertex; a visible one sets its bit in the vertex's NEE block and leaves L to k_nee_resolve
template <bool COUNT, int MINB, bool REALTIME = false, bool NEEAT = false, bool MULTI = false>
__global__ void __launch_bounds__(kTraceThreads, MINB * kTraceCtaScale) k_trace_shadow(const __grid_constant__ LaunchParams p)
{
    uint* ctr = p.wf.counters + p.iteration * kCountersPerIter;
    const uint frontCount = ctr[kCtrShadowCount], count = frontCount + ctr[kCtrShadowShort];      // long rays first (wavefront.cuh: appendShadowRecord)
    if (count == 0) return;
    uint visibleCount = 0, record = 0, slot = 0;
    auto fetchRay = [&](uint i, float3& o, float3& d, float& tMin, float& tMax)
    {
        record = shadowRecordIndex(i, frontCount, MULTI ? neeShadowCapacity(p) : p.wf.capacity);
        const float4 ot = p.wf.shadowOriginTMax[record], dp = p.wf.shadowDirPath[record];
        slot = __float_as_uint(dp.w);
        o = mk3(ot.x, ot.y, ot.z); d = mk3(dp.x, dp.y, dp.z); tMin = 0.0f; tMax = ot.w;
    };
    auto retireRay = [&](uint, const WarpScratch& ws)
    {
        if (uint(ws.bestKey[threadIdx.x & 31u]) != 0xFFFFFFFFu) return;
        // visible: HandleHit's "if any(neeRadianceAndSpecAvg > 0) AccumulatePathRadiance" (PathTracer.hlsli:725-746)
        const uint2 r = p.wf.shadowRadiance[record];
        if constexpr (MULTI) atomicOr(reinterpret_cast<unsigned long long*>(&p.neeBlocks[slot].z), 1ull << r.x);     // `slot`: the block's header, r.x: the sample's index in the block
        else accumulateNeeRadiance<REALTIME>(p, slot, r);
        if constexpr (NEEAT)
        {   // the light was visible: the pixel's feedback reservoir hears about it (PathTracerNEE.hlsli:276-283) and the path's next shade takes the roulette
            // outcome that belongs to a visible sample (shade.cuh)
            const uint4 fb = p.naShadowFeedback[record];
            if (fb.w & 0x80000000u)
            {
                const uint id = p.wf.pixelOfSlot[slot];
                neeat::Reservoir::at(p.na.fbWeight, p.na.fbCandidate, size_t(id & 0xFFFFu) * p.na.W + (id >> 16)).add(__uint_as_float(fb.z), fb.x & 0x7FFFFFFFu, __uint_as_float(fb.y), (fb.x & 0x80000000u) != 0);
                p.naRrFix[slot] = fb.w;
            }
        }
        visibleCount++;
    };
    const TraversalCounters tc = traceLoop<true, COUNT, false, true>(p, ctr + kCtrFetchShadow, count, fetchRay, retireRay);
    if (COUNT) { atomicAdd(ctr + kCtrShadowNodeVisits, tc.nodeVisits); atomicAdd(ctr + kCtrShadowTriTests, tc.triTests); atomicAdd(ctr + kCtrShadowVisible, visibleCount); }
}

// ---- NEE resolve (NEEFullSamples > 1) --------------------------------------------------------------------------------------------------------------
// after k_trace_shadow of the same iteration: one thread per NEE block sums the visible samples in sample order and applies the sum to the path (wavefront.cuh)
template <bool REALTIME>
__global__ void __launch_bounds__(256) k_nee_resolve(const __grid_constant__ LaunchParams p)
{
    const uint count = p.wf.counters[p.iteration * kCountersPerIter + kCtrNeeBlocks];
    const uint stride = 1u + min(kNeeMaxFullSamples, p.c.NEEFullSamples);
    for (uint b = blockIdx.x * blockDim.x + threadIdx.x; b < count; b += gridDim.x * blockDim.x) resolveNeeBlock<REALTIME>(p, p.neeBlocks + size_t(b) * stride);
}

// ---- commit + accumulate ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_commit_accumulate(const __grid_constant__ LaunchParams p)
{
    const uint W = p.c.imageWidth;
    for (uint pix = blockIdx.x * blockDim.x + threadIdx.x; pix < p.wf.pixelCount; pix += gridDim.x * blockDim.x)
    {
        const uint id = p.wf.pixelOfSlot[pix];
        const size_t o = size_t(id & 0xFFFF) * W + (id >> 16);
        float4 acc = p.accumulated[o];
        uint n = p.accumulatedSamples;
        uint2 last = make_uint2(0, 0);
        for (uint s = 0; s < p.subSampleCount; s++)
        {
            const uint2 l = p.radiance[s * p.wf.pixelCount + pix];
            const float r = f16tof32(l.x), g = f16tof32(l.x >> 16), b = f16tof32(l.y);
            last = make_uint2(l.x, (l.y & 0xFFFFu) | (0x3C00u << 16));          // float4(L.rgb, 1) as RGBA16F
            if (p.doAccumulate)
            {   // blend = 1/(n+1); lerp(prev, sample, blend) unless blend >= 1 (Sample.cpp:2775, AccumulationPass.hlsl:57-65)
                const float blend = 1.0f / (float(n) + 1.0f);
                if (blend < 1.0f) { acc.x = acc.x + (r - acc.x) * blend; acc.y = acc.y + (g - acc.y) * blend; acc.z = acc.z + (b - acc.z) * blend; acc.w = acc.w + (1.0f - acc.w) * blend; }
                else acc = make_float4(r, g, b, 1.0f);
                n++;
            }
        }
        p.outputColor[o] = last;
        if (p.doAccumulate) p.accumulated[o] = acc;
    }
}

// ---- standalone ray queries (parity tests, traversal benchmark): the wavefront kernels' traversal loop -------------------------------------
template <bool ANY_HIT>
__global__ void __launch_bounds__(kTraceThreads, 2 * kTraceCtaScale) k_trace_rays(const __grid_constant__ LaunchParams p, const RtxptRay* __restrict__ rays, uint count, RtxptHit* __restrict__ out, uint* counters, uint* cursor)
{
    uint index = 0;
    auto fetchRay = [&](uint i, float3& o, float3& d, float& tMin, float& tMax)
    {
        index = i;
        const float4 a = reinterpret_cast<const float4*>(rays)[i * 2], b = reinterpret_cast<const float4*>(rays)[i * 2 + 1];
        o = mk3(a.x, a.y, a.z); d = mk3(b.x, b.y, b.z); tMin = a.w; tMax = b.w;
    };
    auto retireRay = [&](uint, const WarpScratch& ws)
    {
        uint subInstance; const HitRecord h = Traverser<ANY_HIT, true, false>::result(ws, subInstance);
        RtxptHit r;
        if (h.gid != 0xFFFFFFFFu) { const uint4 info = p.scene.triInfo[h.gid]; r.t = h.t; r.u = h.u; r.v = h.v; r.instanceIndex = info.x; r.geometryIndex = info.y; r.primitiveIndex = info.z; }
        else { r.t = -1.0f; r.u = r.v = 0.f; r.instanceIndex = r.geometryIndex = r.primitiveIndex = 0xFFFFFFFFu; }
        out[index] = r;
    };
    const TraversalCounters tc = traceLoop<ANY_HIT, true, false, false>(p, cursor, count, fetchRay, retireRay);
    if (counters) { atomicAdd(counters + 0, tc.nodeVisits); atomicAdd(counters + 1, tc.triTests); }
}

// ---- tile exchange for multi-GPU (the reference is single-GPU; SURVEY.md §8e) ------------------------------------------------------------------
// pack: owned pixels of the accumulated image -> compact array in slot order; unpack: all ranks' compact arrays -> full frame
__global__ void k_pack_owned(const float4* __restrict__ image, const uint* __restrict__ pixelOfSlot, uint pixelCount, uint paddedCount, uint width, float4* __restrict__ dst)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < paddedCount; i += gridDim.x * blockDim.x)
    {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < pixelCount) { const uint id = pixelOfSlot[i]; v = image[size_t(id & 0xFFFF) * width + (id >> 16)]; }
        dst[i] = v;
    }
}
__global__ void k_unpack_all(const float4* __restrict__ srcAll, const uint* __restrict__ allPixelTable, uint totalEntries, uint width, float4* __restrict__ image)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < totalEntries; i += gridDim.x * blockDim.x)
    {
        const uint id = allPixelTable[i];
        if (id != 0xFFFFFFFFu) image[size_t(id & 0xFFFF) * width + (id >> 16)] = srcAll[i];
    }
}
// generic form for the realtime frame (guides, NRD inputs, output colour): up to kExchangeMaxImages full-frame per-pixel images of 1 / 4 / 8 / 16 bytes per pixel; a rank's block
// holds, image after image, paddedCount elements in slot order (segments start on 16-byte boundaries)
template <typename T> __device__ __forceinline__ void exchangeCopyPack(const ExchangeSet& e, uint k, uint i, uint id, bool owned, uint8_t* dst)
{
    T v{}; if (owned) v = reinterpret_cast<const T*>(e.image[k])[size_t(id & 0xFFFF) * e.width + (id >> 16)];
    reinterpret_cast<T*>(dst + e.segmentOffset[k])[i] = v;
}
__global__ void k_exchange_pack(const __grid_constant__ ExchangeSet e, const uint* __restrict__ pixelOfSlot, uint pixelCount, uint paddedCount, uint8_t* __restrict__ dst)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < paddedCount; i += gridDim.x * blockDim.x)
    {
        const bool owned = i < pixelCount; const uint id = owned ? pixelOfSlot[i] : 0u;
        for (uint k = 0; k < e.count; k++)
            if (e.image[k]) switch (e.bytesPerPixel[k])       // image == NULL: a segment filled by its own kernel (stable-plane neighbour guides)
            {
            case 1: exchangeCopyPack<uint8_t>(e, k, i, id, owned, dst); break;
            case 4: exchangeCopyPack<uint>(e, k, i, id, owned, dst); break;
            case 8: exchangeCopyPack<uint2>(e, k, i, id, owned, dst); break;
            default: exchangeCopyPack<uint4>(e, k, i, id, owned, dst); break;
            }
    }
}
template <typename T> __device__ __forceinline__ void exchangeCopyUnpack(const ExchangeSet& e, uint k, uint slot, uint id, const uint8_t* src)
{
    reinterpret_cast<T*>(e.image[k])[size_t(id & 0xFFFF) * e.width + (id >> 16)] = reinterpret_cast<const T*>(src + e.segmentOffset[k])[slot];
}
__global__ void k_exchange_unpack(const __grid_constant__ ExchangeSet e, const uint* __restrict__ allPixelTable, uint paddedCount, uint world, uint skipRank, const uint8_t* __restrict__ srcAll)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < paddedCount * world; i += gridDim.x * blockDim.x)
    {
        const uint id = allPixelTable[i];
        const uint rank = i / paddedCount, slot = i - rank * paddedCount;
        if (id == 0xFFFFFFFFu || rank == skipRank) continue;                 // the rank's own pixels are already in place
        const uint8_t* src = srcAll + size_t(rank) * e.bytesPerRank;
        for (uint k = 0; k < e.count; k++)
            if (e.image[k]) switch (e.bytesPerPixel[k])
            {
            case 1: exchangeCopyUnpack<uint8_t>(e, k, slot, id, src); break;
            case 4: exchangeCopyUnpack<uint>(e, k, slot, id, src); break;
            case 8: exchangeCopyUnpack<uint2>(e, k, slot, id, src); break;
            default: exchangeCopyUnpack<uint4>(e, k, slot, id, src); break;
            }
    }
}
void launchExchangePack(const ExchangeSet& e, const uint32_t* pixelOfSlot, uint32_t pixelCount, uint32_t paddedCount, void* dst, const GridConfig& g, cudaStream_t s)
{ k_exchange_pack<<<g.smCount * 4, 256, 0, s>>>(e, pixelOfSlot, pixelCount, paddedCount, static_cast<uint8_t*>(dst)); }
void launchExchangeUnpack(const ExchangeSet& e, const uint32_t* allPixelTable, uint32_t paddedCount, uint32_t world, uint32_t skipRank, const void* srcAll, const GridConfig& g, cudaStream_t s)
{ k_exchange_unpack<<<g.smCount * 4, 256, 0, s>>>(e, allPixelTable, paddedCount, world, skipRank, static_cast<const uint8_t*>(srcAll)); }
void launchPackOwned(const float4* image, const uint32_t* pixelOfSlot, uint32_t pixelCount, uint32_t paddedCount, uint32_t width, float4* dst, const GridConfig& g, cudaStream_t s)
{ k_pack_owned<<<g.smCount * 4, 256, 0, s>>>(image, pixelOfSlot, pixelCount, paddedCount, width, dst); }
void launchUnpackAll(const float4* srcAll, const uint32_t* allPixelTable, uint32_t totalEntries, uint32_t width, float4* image, const GridConfig& g, cudaStream_t s)
{ k_unpack_all<<<g.smCount * 4, 256, 0, s>>>(srcAll, allPixelTable, totalEntries, width, image); }

// ---- launch wrappers ---------------------------------------------------------------------------------------------------------------------------
static size_t traceSmemBytes(const LaunchParams& p) { return kTraceScratchBytes + size_t(p.smemNodeCount) * 80; }

// Every wavefront traversal instantiation, one row per TraceKind.  Column 0 counts traversal steps (MINB 2, reference mode only); columns 1..3 are
// MINB 2..4, the resident CTAs per SM the kernel's registers are capped for.  nullptr: no such instantiation.
using TraceKernel = void (*)(LaunchParams);
static const TraceKernel kTraceKernels[][4] = {
    { k_trace_closest<true, 2, true>, k_trace_closest<false, 2, true>,       k_trace_closest<false, 3, true>,  k_trace_closest<false, 4, true> },        // Closest
    { nullptr,                        k_trace_closest<false, 2, false>,      k_trace_closest<false, 3, false>, k_trace_closest<false, 4, false> },       // ClosestRealtime
    { k_trace_shadow<true, 2>,        k_trace_shadow<false, 2>,              k_trace_shadow<false, 3>,         k_trace_shadow<false, 4> },               // Shadow
    { nullptr,                        k_trace_shadow<false, 2, true>,        nullptr,                          k_trace_shadow<false, 4, true> },         // ShadowRealtime
    { nullptr,                        k_trace_shadow<false, 2, false, true>, nullptr,                          k_trace_shadow<false, 4, false, true> },  // ShadowNeeat
    { nullptr,                        k_trace_shadow<false, 2, true, true>,  nullptr,                          k_trace_shadow<false, 4, true, true> },   // ShadowRealtimeNeeat
    { nullptr, k_trace_shadow<false, 2, false, false, true>, nullptr, k_trace_shadow<false, 4, false, false, true> },                                         // ShadowMulti
    { nullptr, k_trace_shadow<false, 2, true, false, true>,  nullptr, k_trace_shadow<false, 4, true, false, true> },                                          // ShadowRealtimeMulti
};
static_assert(sizeof(kTraceKernels) / sizeof(kTraceKernels[0]) == size_t(TraceKind::Count), "one table row per TraceKind");

template <typename K> static cudaError_t allowSmem(K kernel, int bytes) { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); }

cudaError_t configureKernels(int maxSmemOptin)
{
    cudaError_t e;
    const int want = maxSmemOptin > 0 ? maxSmemOptin : 0;
    for (const auto& row : kTraceKernels)
        for (TraceKernel k : row)
            if (k && (e = allowSmem(k, want)) != cudaSuccess) return e;
    if ((e = allowSmem(k_trace_rays<false>, want)) != cudaSuccess) return e;
    return allowSmem(k_trace_rays<true>, want);
}

// launched with the optional L2 access-policy window of GridConfig attached as a per-launch attribute (no stream state is touched)
void launchTrace(TraceKind kind, const LaunchParams& p, const GridConfig& g, bool countSteps, cudaStream_t s)
{
    const TraceKernel* row = kTraceKernels[int(kind)];
    const int minb = std::min(std::max(g.traceBlocksPerSM, 2), 4);
    TraceKernel kernel = row[minb - 1];
    int grid = g.smCount * g.traceBlocksPerSM;
    if (countSteps && row[0]) kernel = row[0];
    else if (!row[2] && minb < 4) { kernel = row[1]; grid = g.smCount * 2; }       // no MINB-3 instantiation: below four CTAs per SM, MINB 2 on two per SM
    cudaLaunchConfig_t cfg = {}; cfg.gridDim = dim3(uint(grid) * kTraceCtaScale); cfg.blockDim = dim3(kTraceThreads); cfg.dynamicSmemBytes = traceSmemBytes(p); cfg.stream = s;
    cudaLaunchAttribute attr[1]; cfg.attrs = attr; cfg.numAttrs = 0;
    if (g.l2WindowBytes)
    {
        attr[0].id = cudaLaunchAttributeAccessPolicyWindow;
        attr[0].val.accessPolicyWindow.base_ptr = const_cast<void*>(g.l2WindowBase); attr[0].val.accessPolicyWindow.num_bytes = g.l2WindowBytes;
        attr[0].val.accessPolicyWindow.hitRatio = g.l2WindowHitRatio;
        attr[0].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting; attr[0].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cfg.numAttrs = 1;
    }
    cudaLaunchKernelEx(&cfg, kernel, p);
}

void launchGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_generate<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchCommitAccumulate(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_commit_accumulate<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchNeeResolve(const LaunchParams& p, const GridConfig& g, bool realtime, cudaStream_t s)
{
    if (realtime) k_nee_resolve<true><<<g.smCount * 4, 256, 0, s>>>(p); else k_nee_resolve<false><<<g.smCount * 4, 256, 0, s>>>(p);
}
void launchTraceRays(const LaunchParams& p, const GridConfig& g, const RtxptRay* rays, uint32_t count, bool anyHit, RtxptHit* out, uint32_t* counters, uint32_t* cursor, cudaStream_t s)
{
    cudaMemsetAsync(cursor, 0, sizeof(uint32_t), s);
    if (anyHit) k_trace_rays<true><<<g.smCount * g.traceBlocksPerSM * kTraceCtaScale, kTraceThreads, traceSmemBytes(p), s>>>(p, rays, count, out, counters, cursor);
    else k_trace_rays<false><<<g.smCount * g.traceBlocksPerSM * kTraceCtaScale, kTraceThreads, traceSmemBytes(p), s>>>(p, rays, count, out, counters, cursor);
}

} // namespace pt
