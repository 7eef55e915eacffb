// realtime_kernels.cu — realtime mode (stable planes) on the wavefront of kernels.cu.  One call of rtxpt_b200_path_trace_realtime replaces the
// reference's three kinds of dispatch (Rtxpt/Sample.cpp:2455-2521, Rtxpt/Shaders/PathTracerSample.hlsl:201-232):
//   BUILD  k_rt_build_generate -> [ k_trace_closest -> k_rt_shade<BUILD> ]*      RayGen with PATH_TRACER_MODE_BUILD_STABLE_PLANES: delta-only exploration,
//          one branch of a pixel's delta tree at a time (postProcessHit, PathTracerSample.hlsl:96-113); no NEE, no Russian roulette, no shadow rays
//   FILL   per sub-sample: k_rt_fill_generate (FirstHitFromVBuffer, PathTracerSample.hlsl:33-93) -> [ k_trace_closest -> k_rt_shade<FILL> ->
//          k_trace_shadow<realtime> ]* -> k_rt_fill_commit (CommitPixel = CommitDenoiserRadiance)
//   MERGE  k_rt_merge: PostProcess NO_DENOISER_FINAL_MERGE (ProcessingPasses/PostProcess.hlsl:692-709) = StablePlanesContext::GetAllRadiance
// Sub-samples run one after the other like the reference's back-to-back dispatches: each adds to the fp16 radiance of the plane records, and the
// order of those additions is part of the result.  Compiled with the shade unit's flags (fast-math in the default build, IEEE in the strict one).
#if !RTXPT_STRICT_FP
#define PT_FAST_MATH 1
#endif
// (the Sobol byte tables of shade_kernels.cu are private to that unit; this one evaluates the direction numbers bit by bit - same values)
#include "shade.cuh"
#include "guides_filter.cuh"
#include "denoiser_iface.cuh"
#include "kernels.h"

namespace pt {

PT_DEVICE void appendRay(uint* queue, uint* counter, bool valid, uint entry)
{
    const uint lane = threadIdx.x & 31u;
    const uint peers = __ballot_sync(0xFFFFFFFFu, valid);
    if (valid)
    {
        const uint leader = __ffs(peers) - 1u;
        uint base = 0;
        if (lane == leader) base = atomicAdd(counter, __popc(peers));
        base = __shfl_sync(peers, base, leader);
        queue[base + __popc(peers & ((1u << lane) - 1u))] = entry;
    }
}

// ---- BUILD: EmptyPathInitialize + StartPixel (PathTracer.hlsli:47-113) -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rt_build_generate(const __grid_constant__ LaunchParams p)
{
    const uint total = p.wf.pixelCount;
    if (blockIdx.x == 0 && threadIdx.x == 0) p.wf.counters[kCtrRayCount] = total;
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < total; slot += gridDim.x * blockDim.x)
    {
        const uint id = p.wf.pixelOfSlot[slot];
        PathRegs path;
        path.id = id; path.sceneLength = 0.f;
        path.flagsAndVertexIndex = 0; path.packedCounters = 0; path.interior0 = path.interior1 = 0;
        path.setThp(mk3(1.f));
        path.setFlag(kPFActive, true); path.setFlag(kPFDeltaOnlyPath, true);
        path.setCone(0.f, p.c.camera.PixelConeSpreadAngle);
        Mat3 ident; ident.r0 = mk3(1, 0, 0); ident.r1 = mk3(0, 1, 0); ident.r2 = mk3(0, 0, 1);
        packOrthoMatrix(ident, path.lXY, path.lZW);                    // SetImageXform(identity)
        path.setFlag(kPFStablePlaneOnDominantBranch, true);
        path.pack0 = __float_as_uint(0.0f); path.pack1 = 0;            // SetMotionVectorSceneLength(0)
        path.setStablePlaneIndex(0);
        path.stableBranchID() = 1;
        if (hasFinishedSurfaceBounces(p.c, 1, 0)) path.setFlag(kPFTerminateAtNextBounce, true);
        float3 origin, dir; computeCameraRay(p.c, id, p.firstSampleIndex, origin, dir);
        path.origin = origin; path.dir = dir;
        // StablePlanesContext::StartPixel + Bridge::ExportSurfaceInit
        const size_t o = pixelOffset(p, id);
        p.rt.stableRadiance[o] = make_uint2(0u, 0u);
        headerWord(p, id, 0) = kInvalidBranchID; headerWord(p, id, 1) = kInvalidBranchID; headerWord(p, id, 2) = kInvalidBranchID;
        p.depth[o] = 0.0f; p.rt.specularHitT[o] = 0.0f;
        path.store(p.wf, slot);
        p.wf.rayQueue[0][slot] = slot | (path.hasFlag(kPFTerminateAtNextBounce) ? 0x80000000u : 0u);
    }
}

// ---- FILL: EmptyPathInitialize + FirstHitFromVBuffer(path, 0) ------------------------------------------------------------------------------------------
// The reference narrows the first ray to [0.99, 1.01] x the stored hit distance "for performance reasons"; the ray is the one the BUILD pass
// traced, so its closest hit over [0, inf) is the same hit and the interval is left open here.
__global__ void __launch_bounds__(256) k_rt_fill_generate(const __grid_constant__ LaunchParams p)
{
    const uint total = p.wf.pixelCount;
    uint* ctr = p.wf.counters;
    for (uint base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; base < total; base += gridDim.x * blockDim.x)
    {
        const uint slot = base + (threadIdx.x & 31u);
        bool queued = false; uint entry = 0;
        if (slot < total)
        {
            const uint id = p.wf.pixelOfSlot[slot];
            PathRegs path;
            path.id = id; path.sceneLength = 0.f;
            path.flagsAndVertexIndex = 0; path.packedCounters = 0; path.interior0 = path.interior1 = 0;
            path.setFlag(kPFActive, true); path.setFlag(kPFDeltaOnlyPath, true);
            path.setCone(0.f, p.c.camera.PixelConeSpreadAngle);
            path.setL(make_float4(0.f, 0.f, 0.f, 0.f));
            path.setFireflyK_BsdfPdf(1.0f, 0.0f);
            path.setMisInfo_RuRu(0u, 1.0f);
            const uint4* rec = reinterpret_cast<const uint4*>(p.rt.planes + planeAddress(p.rt, id, 0));
            const uint4 r0 = rec[0], r1 = rec[1], r2 = rec[2];
            float sceneLength = __uint_as_float(r1.w); const float lastRayT = __uint_as_float(r0.w);
            const uint vertexIndex = r2.w >> 16;
            bool isMiss = false;
            if (!isfinite(sceneLength)) { sceneLength = kMaxRayTravel; isMiss = true; } else sceneLength -= lastRayT;
            path.setVertexIndex(vertexIndex - 1);
            path.origin = mk3(__uint_as_float(r0.x), __uint_as_float(r0.y), __uint_as_float(r0.z));
            path.dir = mk3(__uint_as_float(r1.x), __uint_as_float(r1.y), __uint_as_float(r1.z));
            path.setFlag(kPFStablePlaneOnPlane, true); path.setFlag(kPFStablePlaneOnBranch, true);
            path.setStablePlaneIndex(0);
            path.stableBranchID() = headerWord(p, id, 0);
            path.setThp(mk3(f16tof32(r2.x >> 16), f16tof32(r2.y >> 16), f16tof32(r2.z >> 16)));
            path.setFlag(kPFStablePlaneOnDominantBranch, (headerWord(p, id, 3) & 3u) == 0u);
            path.setCounter(kCtrBouncesFromStablePlane, 0);
            if (hasFinishedSurfaceBounces(p.c, path.vertexIndex() + 1, path.counter(kCtrDiffuseBounces))) path.setFlag(kPFTerminateAtNextBounce, true);
            {   // UpdatePathTravelledLengthOnly(path, sceneLength)
                const float angle = path.coneSpread(), width = path.coneWidth();
                path.setCone(angle * sceneLength + width, angle);
                path.sceneLength = fminf(path.sceneLength + sceneLength, kMaxRayTravel);
            }
            if (isMiss) shadeMiss<false, kModeFillStablePlanes>(p, path);       // inline miss shader: the sky was captured by the BUILD pass, the path just ends
            path.store(p.wf, slot);
            queued = path.hasFlag(kPFActive);
            entry = slot | (path.hasFlag(kPFTerminateAtNextBounce) ? 0x80000000u : 0u);
        }
        appendRay(p.wf.rayQueue[0], ctr + kCtrRayCount, queued, entry);
    }
}

// ---- shade ------------------------------------------------------------------------------------------------------------------------------------------------------
#ifndef PT_RT_SHADE_CTAS
#define PT_RT_SHADE_CTAS 4      // resident CTAs of 128 threads per SM: 4 caps the shade kernels at 128 registers (a few dozen bytes of spills), 3 lets them run without spills.
                                // H100 SXM (700 W): config-3 trace 41.5 ms/frame with 4, 42.4 with 3; the 1-spp realtime frame 9.69 ms with 4, 9.60 with 3
#endif
// MULTI (FILL pass, NEEFullSamples > 1): shadeHit appends the vertex's shadow records and NEE block itself, one record per valid light sample; 3 CTAs per SM, which
// lets it run without spills in both builds.  AMIS (FILL pass): approximate light-vs-BSDF MIS; the BUILD pass evaluates no MIS (PathState.hlsli:157-159) and has one kernel for both kinds
// STF: stochastic texture filtering of the material fetches (rtxpt_b200_set_texture_filtering); its kernels carry analytic lights, gated by the light type at run time
// DEBUG_VIEW (BUILD pass): a first-hit debug view is set (rtxpt_b200_set_debug_view); its kernels carry analytic lights, gated by the light type at run time
template <int MODE, bool ANALYTIC_LIGHTS, bool NEEAT = false, bool MULTI = false, bool AMIS = false, bool STF = false, bool DEBUG_VIEW = false>
__global__ void __launch_bounds__(128, (MULTI || STF) ? 3 : PT_RT_SHADE_CTAS) k_rt_shade(const __grid_constant__ LaunchParams p)
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
        for (uint base = warpGlobal * 32u; base < count; base += warpStride * 32u)
        {
            const uint i = base + lane;
            bool continues = false, shadow = false; uint rayEntry = 0;
            HitOutputs out; out.continuePath = false; out.emitShadow = false;
            if (i < count)
            {
                const uint slot = queue[i];
                PathRegs path; path.load(p.wf, slot, true);
                if constexpr (NEEAT) out.naRecord = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
                if (cls == 0) shadeMiss<false, MODE, NEEAT, AMIS>(p, path);
                else shadeHit<false, ANALYTIC_LIGHTS, MODE, NEEAT, MULTI, AMIS, STF, DEBUG_VIEW>(p, path, slot, p.wf.hits[slot], out);
                continues = (cls != 0) && out.continuePath;
                if constexpr (MODE == kModeBuildStablePlanes)
                {   // postProcessHit: when this branch has ended, continue with the next enqueued branch of the pixel (planes above the current one)
                    if (!continues)
                    {
                        const uint id = path.id;
                        for (uint next = path.stablePlaneIndex() + 1; next < kStablePlaneCount; next++)
                            if (headerWord(p, id, next) == kEnqueuedBranchID) { explorationStart(p, path, id, next); continues = true; break; }
                    }
                }
                path.store(p.wf, slot);         // the commit kernel reads the whole state (plane index, L) of ended paths too
                if (continues) rayEntry = slot | (path.hasFlag(kPFTerminateAtNextBounce) ? 0x80000000u : 0u);
                shadow = out.emitShadow;
            }
            appendRay(nextQueue, ctrNext + kCtrRayCount, continues, rayEntry);
            if constexpr (MODE == kModeFillStablePlanes && !MULTI)
            {
                const uint b = appendShadowRecord(p, ctr, shadow, out.shadow.originTMax.w);
                if (shadow)
                {
                    p.wf.shadowOriginTMax[b] = out.shadow.originTMax; p.wf.shadowDirPath[b] = out.shadow.dirPath; p.wf.shadowRadiance[b] = out.shadow.radiance;
                    if constexpr (NEEAT) p.naShadowFeedback[b] = out.naRecord;
                }
            }
        }
    }
}

// ---- FILL: CommitPixel ----------------------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rt_fill_commit(const __grid_constant__ LaunchParams p)
{
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x)
    {
        PathRegs path; path.load(p.wf, slot, true);
        commitDenoiserRadiance(p, path);
    }
}

// ---- no-denoiser merge: u_OutputColor = float4(stable radiance + noisy radiance of every valid plane, 1) ------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rt_merge(const __grid_constant__ LaunchParams p)
{
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x)
    {
        const uint id = p.wf.pixelOfSlot[slot];
        const size_t o = pixelOffset(p, id);
        const uint2 sr = p.rt.stableRadiance[o];
        float3 L = mk3(f16tof32(sr.x), f16tof32(sr.x >> 16), f16tof32(sr.y));
        for (uint i = 0; i < kStablePlaneCount; i++)
        {
            if (headerWord(p, id, i) == kInvalidBranchID) continue;
            const uint2 n = *(reinterpret_cast<const uint2*>(p.rt.planes + planeAddress(p.rt, id, i)) + 8);
            L = L + mk3(f16tof32(n.x), f16tof32(n.x >> 16), f16tof32(n.y));
        }
        p.outputColor[o] = make_uint2(f32tof16(L.x) | (f32tof16(L.y) << 16), f32tof16(L.z) | (0x3C00u << 16));
    }
}

// ---- StablePlanesDebugViz (PathTracerDebug.hlsli:359-461), run after the FILL passes (Sample.cpp:2551-2555): one thread per pixel of the context ---------------------------
struct DebugVizBuffers
{
    const LaunchParams& p;
    __device__ uint branchID(uint x, uint y, uint plane) const { return headerWord(p, (x << 16) | y, plane); }
    __device__ RtxptStablePlane plane(uint x, uint y, uint plane) const { return p.rt.planes[planeAddress(p.rt, (x << 16) | y, plane)]; }
    __device__ uint dominantIndex(uint x, uint y) const { return headerWord(p, (x << 16) | y, 3) & 3u; }
    __device__ float3 stableRadiance(uint x, uint y) const { const uint2 r = p.rt.stableRadiance[size_t(y) * p.c.imageWidth + x]; return mk3(f16tof32(r.x), f16tof32(r.x >> 16), f16tof32(r.y)); }
};
__global__ void __launch_bounds__(256) k_rt_debug_viz(const __grid_constant__ LaunchParams p)
{
    const DebugVizBuffers buffers{ p };
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x)
    {
        const uint id = p.wf.pixelOfSlot[slot];
        const float4 c = stablePlaneDebugPixel(p.dbg.view, p.dbg.planeIndex, id >> 16, id & 0xFFFFu, p.c.imageWidth, p.c.imageHeight, buffers);      // the split reads other pixels' planes
        if (c.w > 0.0f) p.dbg.viz[pixelOffset(p, id)] = packDebugPixel(c);
    }
}

// ---- RTXPT's side of the denoiser interface (SURVEY §8 row a18): bodies in denoiser_iface.cuh ----
__global__ void __launch_bounds__(256) k_dn_prepare_inputs(const __grid_constant__ LaunchParams p)
{
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x) dnPrepareInputsPixel(p, p.wf.pixelOfSlot[slot]);
}
// DEBUG_VIEW: a denoiser-merge debug view is set (rtxpt_b200_set_debug_view); the merge also draws it
template <bool DEBUG_VIEW = false>
__global__ void __launch_bounds__(256) k_dn_final_merge(const __grid_constant__ LaunchParams p)
{
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x)
    {
        dnFinalMergePixel(p, p.wf.pixelOfSlot[slot]);
        if constexpr (DEBUG_VIEW) dnFinalMergeDebugPixel(p, p.wf.pixelOfSlot[slot]);
    }
}
// DENOISER_DLSS_RR: one thread per owned pixel; the DLSS-RR targets are an argument of their own (denoiser_iface.cuh)
__global__ void __launch_bounds__(256) k_dn_prepare_dlss_rr(const __grid_constant__ LaunchParams p, const DlssRrTargets rr)
{
    for (uint slot = blockIdx.x * blockDim.x + threadIdx.x; slot < p.wf.pixelCount; slot += gridDim.x * blockDim.x) dnPrepareDlssRrPixel(p, rr, p.wf.pixelOfSlot[slot]);
}
// DenoiseSpecHitT: one thread per pixel over the full frame (row-major guides); src / dst alternate between the guide and a scratch image
__global__ void __launch_bounds__(256) k_dn_spec_hitt(const float* __restrict__ src, const float* __restrict__ depth, float* __restrict__ dst, int W, int H)
{
    const int x = int(blockIdx.x * 16 + threadIdx.x), y = int(blockIdx.y * 16 + threadIdx.y);
    if (x < W && y < H) dst[size_t(y) * W + x] = specHitTNeighbourhood(src, depth, W, H, x, y);
}
// multi-GPU (SURVEY §8e): what ComputeDisocclusionRelaxation reads of a pixel's four neighbours - per plane the branch ID (header layer) and the packed plane normal - travels
// with the guides, 24 bytes per pixel: segment layout [plane][word][slot], word 0 = branch ID, word 1 = PackedNormal
__global__ void __launch_bounds__(256) k_rt_pack_plane_guides(const __grid_constant__ LaunchParams p, uint paddedCount, uint* __restrict__ dst)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < paddedCount; i += gridDim.x * blockDim.x)
    {
        const bool owned = i < p.wf.pixelCount; const uint id = owned ? p.wf.pixelOfSlot[i] : 0u;
        for (uint plane = 0; plane < kStablePlaneCount; plane++)
        {
            uint branch = kInvalidBranchID, normal = 0u;
            if (owned) { branch = headerWord(p, id, plane); normal = p.rt.planes[planeAddress(p.rt, id, plane)].PackedNormal; }
            dst[size_t(plane * 2 + 0) * paddedCount + i] = branch; dst[size_t(plane * 2 + 1) * paddedCount + i] = normal;
        }
    }
}
__global__ void __launch_bounds__(256) k_rt_unpack_plane_guides(const __grid_constant__ LaunchParams p, const uint* __restrict__ allPixelTable, uint paddedCount, uint world, uint skipRank, const uint8_t* __restrict__ srcAll,
                                                                size_t segmentOffset, size_t bytesPerRank)
{
    for (uint i = blockIdx.x * blockDim.x + threadIdx.x; i < paddedCount * world; i += gridDim.x * blockDim.x)
    {
        const uint id = allPixelTable[i]; const uint rank = i / paddedCount, slot = i - rank * paddedCount;
        if (id == 0xFFFFFFFFu || rank == skipRank) continue;
        const uint* src = reinterpret_cast<const uint*>(srcAll + size_t(rank) * bytesPerRank + segmentOffset);
        for (uint plane = 0; plane < kStablePlaneCount; plane++)
        {
            headerWord(p, id, plane) = src[size_t(plane * 2 + 0) * paddedCount + slot];
            p.rt.planes[planeAddress(p.rt, id, plane)].PackedNormal = src[size_t(plane * 2 + 1) * paddedCount + slot];
        }
    }
}
void launchRtPackPlaneGuides(const LaunchParams& p, uint32_t paddedCount, void* dst, const GridConfig& g, cudaStream_t s) { k_rt_pack_plane_guides<<<g.smCount * 4, 256, 0, s>>>(p, paddedCount, static_cast<uint*>(dst)); }
void launchRtUnpackPlaneGuides(const LaunchParams& p, const uint32_t* allPixelTable, uint32_t paddedCount, uint32_t world, uint32_t skipRank, const void* srcAll, size_t segmentOffset, size_t bytesPerRank, const GridConfig& g, cudaStream_t s)
{ k_rt_unpack_plane_guides<<<g.smCount * 4, 256, 0, s>>>(p, allPixelTable, paddedCount, world, skipRank, static_cast<const uint8_t*>(srcAll), segmentOffset, bytesPerRank); }
void launchDnSpecHitT(const float* src, const float* depth, float* dst, int W, int H, cudaStream_t s) { k_dn_spec_hitt<<<dim3((W + 15) / 16, (H + 15) / 16), dim3(16, 16), 0, s>>>(src, depth, dst, W, H); }
void launchDnPrepareInputs(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_dn_prepare_inputs<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchDnPrepareDlssRr(const LaunchParams& p, const DlssRrTargets& rr, const GridConfig& g, cudaStream_t s) { k_dn_prepare_dlss_rr<<<g.smCount * 4, 256, 0, s>>>(p, rr); }
void launchDnFinalMerge(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    if (p.dbg.viz && isDenoiserMergeView(p.dbg.view)) k_dn_final_merge<true><<<g.smCount * 4, 256, 0, s>>>(p); else k_dn_final_merge<<<g.smCount * 4, 256, 0, s>>>(p);
}

void launchRtBuildGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_rt_build_generate<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchRtFillGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_rt_fill_generate<<<g.smCount * 4, 256, 0, s>>>(p); }
template <bool AMIS>
static void launchRtShadeNeeatMis(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    const int grid = g.smCount * PT_RT_SHADE_CTAS;
    if (p.stf.pointTextures) { k_rt_shade<kModeFillStablePlanes, true, true, false, AMIS, true><<<g.smCount * 3, 128, 0, s>>>(p); return; }
    if (p.scene.analyticLightCount != 0) k_rt_shade<kModeFillStablePlanes, true, true, false, AMIS><<<grid, 128, 0, s>>>(p); else k_rt_shade<kModeFillStablePlanes, false, true, false, AMIS><<<grid, 128, 0, s>>>(p);
}
void launchRtShadeNeeat(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{   // FILL pass with NEE-AT feedback: tile-sampler candidates, MIS against the global table, feedback records for the shadow kernel
    if (p.c.useApproximateMIS) launchRtShadeNeeatMis<true>(p, g, s); else launchRtShadeNeeatMis<false>(p, g, s);
}
template <bool AMIS>
static void launchRtShadeFill(const LaunchParams& p, const GridConfig& g, cudaStream_t s)
{
    const int grid = g.smCount * PT_RT_SHADE_CTAS;
    if (p.stf.pointTextures)
    {
        if (min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1) k_rt_shade<kModeFillStablePlanes, true, false, true, AMIS, true><<<g.smCount * 3, 128, 0, s>>>(p);
        else k_rt_shade<kModeFillStablePlanes, true, false, false, AMIS, true><<<g.smCount * 3, 128, 0, s>>>(p);
        return;
    }
    if (min(kNeeMaxFullSamples, p.c.NEEFullSamples) > 1) k_rt_shade<kModeFillStablePlanes, true, false, true, AMIS><<<g.smCount * 3, 128, 0, s>>>(p);      // several light samples per vertex: analytic lights gated at run time
    else { if (p.scene.analyticLightCount != 0) k_rt_shade<kModeFillStablePlanes, true, false, false, AMIS><<<grid, 128, 0, s>>>(p); else k_rt_shade<kModeFillStablePlanes, false, false, false, AMIS><<<grid, 128, 0, s>>>(p); }
}
void launchRtShade(const LaunchParams& p, const GridConfig& g, bool fill, cudaStream_t s)
{
    const int grid = g.smCount * PT_RT_SHADE_CTAS;
    if (!fill && p.dbg.viz && isFirstHitView(p.dbg.view))
    {   // first-hit debug view: drawn by the BUILD pass, whose vertex 1 is the camera ray's hit
        if (p.stf.pointTextures) k_rt_shade<kModeBuildStablePlanes, true, false, false, false, true, true><<<g.smCount * 3, 128, 0, s>>>(p);
        else k_rt_shade<kModeBuildStablePlanes, true, false, false, false, false, true><<<grid, 128, 0, s>>>(p);
        return;
    }
    if (!fill && p.stf.pointTextures) { k_rt_shade<kModeBuildStablePlanes, true, false, false, false, true><<<g.smCount * 3, 128, 0, s>>>(p); return; }
    if (!fill) { if (p.scene.analyticLightCount != 0) k_rt_shade<kModeBuildStablePlanes, true><<<grid, 128, 0, s>>>(p); else k_rt_shade<kModeBuildStablePlanes, false><<<grid, 128, 0, s>>>(p); }
    else if (p.c.useApproximateMIS) launchRtShadeFill<true>(p, g, s);
    else launchRtShadeFill<false>(p, g, s);
}
void launchRtFillCommit(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_rt_fill_commit<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchRtMerge(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_rt_merge<<<g.smCount * 4, 256, 0, s>>>(p); }
void launchRtDebugViz(const LaunchParams& p, const GridConfig& g, cudaStream_t s) { k_rt_debug_viz<<<g.smCount * 4, 256, 0, s>>>(p); }

} // namespace pt
