// wavefront.cuh — per-path state in HBM (structure of arrays), queues and launch parameters of the wavefront path tracer.
//
// The reference keeps an 80-byte PathState in the DXR payload of a megakernel (Rtxpt/Shaders/PathTracer/PathState.hlsli:83-121,
// PathPayload.hlsli:19-27).  Here the same 80 bytes live in five uint4 arrays (structure of arrays), so that every kernel of the
// wavefront reads/writes whole 16-byte words that are contiguous across a warp whenever the indices are:
//   s0: origin.xyz, id            s1: dir.xyz, sceneLength          s2: thp(fp16 x4), L(fp16 x4)   (reference mode: thp, h, 0)
//   s3: interiorList[0..1], packedCounters, rayCone(fp16 x2)        s4: fireflyK|bsdfPdf, misInfo|ruRuCorrection, flagsAndVertexIndex, sampleIndex
// (stableBranchID of the reference payload is unused in reference mode; its word carries the path's sample index instead.)
//
// Reference mode keeps the state in ray order: iteration i's rays are entries 0..count-1 of state set i & 1 (LaunchParams::stateIn), and
// k_shade appends each continuing path to the other set (stateOut) with a warp-aggregated counter, so the ray index is the position and
// every kernel reads and writes the state in whole, contiguous sectors.  Only the radiance stays at the path's home index
// h = sub-sample * pixelCount + pixel slot (LaunchParams::radiance, fp16 x4): the shadow kernel adds to it while the next iteration's
// closest-hit kernel already runs, and the commit kernel reads it per pixel.  s2 carries h in place of L, and s1.w carries
// kPFTerminateAtNextBounce in its sign bit (sceneLength is never negative) so that the closest-hit kernel bins terminating paths from the
// words it reads anyway.  Realtime mode indexes one state set by path slot through its ray queues.
#pragma once
#include "device_math.cuh"
#include "neeat.cuh"
#include "scene_device.cuh"

namespace pt {

constexpr int kNumShadeClasses = 6;     // 0 miss, 1 hit on a path that terminates at this vertex, 2..5 material classes (SER sort key analogue)
constexpr int kMaxWavefrontIterations = 64;   // reference mode needs bounceCount + 5; the BUILD pass of realtime mode explores up to three delta branches per pixel one after the other

struct ShadowRecord         // 40 bytes in three arrays
{
    float4 originTMax;      // ComputeVisibilityRay origin, shortened tMax
    float4 dirPath;         // direction, path slot (realtime) or home index h (reference mode) as bits
    uint2  radiance;        // NEEResult::RadianceAndSpecAvgPkg (fp16 x4): what L gains if the light is visible
};

struct StateSet { uint4* s0; uint4* s1; uint4* s2; uint4* s3; uint4* s4; };

struct WavefrontBuffers
{
    uint4* s0; uint4* s1; uint4* s2; uint4* s3; uint4* s4;     // realtime mode's state, per path slot (reference mode: state set 0)
    float4* hits;                   // t,u,v,gid per path slot (reference mode: per ray)
    uint* rayQueue[2];              // realtime mode: path slots whose scatter ray is to be traced (ping-pong per iteration)
    uint* shadeQueue;               // kNumShadeClasses regions of `capacity` entries: ray indices (reference mode) or path slots (realtime)
    float4* shadowOriginTMax; float4* shadowDirPath; uint2* shadowRadiance;
    uint* counters;                 // see Counter* below, one block per iteration
    const uint* pixelOfSlot;        // packed (x<<16)|y of the pixels this context renders (tile partition), per pixel slot
    uint capacity;                  // path slots
    uint pixelCount;                // pixels rendered by this context
};

// counters layout: per iteration i a block of kCountersPerIter uints
constexpr int kCtrRayCount = 0;                 // rays queued for iteration i
constexpr int kCtrShadeCount = 1;               // + class
constexpr int kCtrShadowCount = 1 + kNumShadeClasses;
constexpr int kCtrNodeVisits = kCtrShadowCount + 1;         // closest-hit traversal (instrumented builds only)
constexpr int kCtrTriTests = kCtrNodeVisits + 1;
constexpr int kCtrShadowVisible = kCtrTriTests + 1;
constexpr int kCtrShadowNodeVisits = kCtrShadowVisible + 1;  // any-hit traversal
constexpr int kCtrShadowTriTests = kCtrShadowNodeVisits + 1;
constexpr int kCtrFetchClosest = kCtrShadowTriTests + 1;    // dynamic ray fetch cursors of the persistent traversal warps
constexpr int kCtrFetchShadow = kCtrFetchClosest + 1;
constexpr int kCtrShadowShort = kCtrFetchShadow + 1;        // shadow records appended from the END of the record arrays (see appendShadowRecord); kCtrShadowCount counts the ones at the front
constexpr int kCtrNeeBlocks = kCtrShadowShort + 1;          // NEE blocks appended by a multi-sample shade (NEEFullSamples > 1, see NEE blocks below)
static_assert(kCtrNeeBlocks < 20, "counter block");
constexpr int kCountersPerIter = 20;

// realtime mode (stable planes): the reference's u_StablePlanesHeader / u_StablePlanesBuffer / u_StableRadiance / u_SpecularHitT and the
// realtime fields of PathTracerConstants (StablePlanes.hlsli:82-274, PathTracerShared.h:57-80)
struct RealtimeParams
{
    RtxptStablePlane* planes;       // [3 * planeStride], GenericTS addressing
    uint* header;                   // [4][height][width]
    uint2* stableRadiance;          // RGBA16F
    float* specularHitT;
    uint lineStride, planeStride;
    uint activePlaneCount, maxVertexDepth, allowPSR;
    float attenuation;              // invSubSampleCount
    float worldToClipNoOffset[16], prevWorldToClipNoOffset[16];
    float clipToWindowScale[2];
    // denoiser interface (PostProcess.hlsl DENOISER_PREPARE_INPUTS / DENOISER_FINAL_MERGE)
    float* dnViewZ; uint2* dnMotion; uint* dnNormalRoughness; uint2* dnDiff; uint2* dnSpec; unsigned char* dnDisocclusionMix; unsigned char* dnHistoryClampRelax;
    const uint2* dnDenoisedDiff; const uint2* dnDenoisedSpec;
    RtxptDenoiserConstants dn; uint dnPlane, dnInitWithStableRadiance;
};

struct LaunchParams;
// Shadow records are appended from both ends of the record arrays: rays with a long way to go (tMax above LaunchParams::shadowLongRayT: environment and far-light samples,
// which walk most of the scene when nothing blocks them) at the front, the rest from the back.  The persistent any-hit kernel fetches front to back, so the longest traversals of a
// launch start first and its tail - one warp finishing a 100+ node walk while 147 SMs idle - overlaps the bulk of the short rays (longest-processing-time-first).  Index of a record:
PT_DEVICE uint shadowRecordIndex(uint i, uint frontCount, uint capacity) { return i < frontCount ? i : capacity - 1u - (i - frontCount); }

struct LaunchParams
{
    SceneView scene;
    WavefrontBuffers wf;
    RtxptPathTracerConstants c;
    uint firstSampleIndex;          // sampleBaseIndex + firstSubSampleIndex
    uint subSampleCount;
    uint iteration;
    uint smemNodeCount;             // BVH nodes staged in shared memory
    uint flags;
    int refillThreshold;            // dynamic fetch: a warp refills its idle lanes when fewer than this many lanes are still traversing
    int waitFlushLanes;             // a partial group of triangle tests is drained once this many lanes wait for nothing but their results
    float shadowLongRayT;           // shadow rays with tMax above this are queued at the front (a quarter of the scene diagonal)
    // render targets
    uint2* outputColor;             // RGBA16F, full frame, last sub-sample
    float4* accumulated;            // RGBA32F, full frame
    float* depth;                   // guide buffers (RTXPT_CFG_EXPORT_GUIDES): R32F depth, RGBA16F motion vectors, R11G11B10 throughput
    uint2* motionVectors; uint* throughput;
    float worldToClip[16];          // view.matWorldToClip, row-major, row vector x matrix
    uint exportGuides;
    uint accumulatedSamples;        // before this call
    uint doAccumulate;
    RealtimeParams rt;
    // NEE-AT temporal feedback (kernels instantiated with NEEAT = true only; appended so that every other kernel's parameter offsets stay what they were)
    neeat::Params na;
    union
    {
        uint4* naShadowFeedback;    // per shadow record: light | ssc << 31, feedback weight, reservoir random, Russian roulette outcome had the sample been visible
        uint4* neeBlocks;           // NEEFullSamples > 1 (multi-sample kernels, which never run with feedback): the NEE blocks (see below)
    };
    uint* naRrFix;                  // per home index h: set by the shadow kernel when the sample was visible, consumed by the next shade of the path
    // reference mode's ray-ordered state (see the top of this file; appended for the same reason): the set this iteration's rays are read from,
    // the set its continuing paths are appended to, and the radiance per home index h
    StateSet stateIn, stateOut;
    uint2* radiance;
};
static_assert(sizeof(LaunchParams) == 1632, "the parameter block of every kernel keeps its layout");

// ---- NEE blocks (NEEFullSamples = N > 1) ---------------------------------------------------------------------------------------------------------------
// A vertex that takes light samples appends one block of 1 + N uint4 (counter kCtrNeeBlocks) to LaunchParams::neeBlocks: a header { path slot or home index h, the FILL
// pass's specular-average choice bits (shade.cuh), visibility mask bits 0..31, bits 32..63 } and per sample j the fp32 (radiance.rgb, specAvg) it adds if visible.  The
// shadow-record arrays then hold up to N records per path: sample j's record carries the header's index in dirPath.w and j in radiance.x; the shadow kernel sets bit j
// of the mask when the light is visible, and k_nee_resolve sums the block.
constexpr uint kNeeMaxFullSamples = 63;         // min( 63, NEEFullSamples ), PathTracerNEE.hlsli:306
PT_HD uint neeShadowCapacity(const LaunchParams& p) { return p.wf.capacity * min(kNeeMaxFullSamples, p.c.NEEFullSamples); }      // length of the shadow-record arrays

// warp-aggregated append of one entry per calling lane among the lanes that are active together (the multi-sample shade appends from inside its divergent sample loop)
PT_DEVICE uint appendActive(uint* ctr)
{
#ifdef __CUDA_ARCH__
    const uint active = __activemask(), lane = threadIdx.x & 31u, leader = __ffs(active) - 1u;
    uint base = 0;
    if (lane == leader) base = atomicAdd(ctr, __popc(active));
    return __shfl_sync(active, base, leader) + __popc(active & ((1u << lane) - 1u));
#else
    return atomicAdd(ctr, 1u);      // host build of the shading functions (tests/emu): one lane
#endif
}
// appendShadowRecord for the lanes that are active together, every one of which emits a record; `capacity` is the length of the record arrays
PT_DEVICE uint appendShadowRecordActive(const LaunchParams& p, uint* ctr, float tMax, uint capacity)
{
    const bool isLong = tMax > p.shadowLongRayT;
#ifdef __CUDA_ARCH__
    const uint active = __activemask(), lane = threadIdx.x & 31u;
    const uint longPeers = __ballot_sync(active, isLong), peers = isLong ? longPeers : (active & ~longPeers), leader = __ffs(peers) - 1u;
    uint base = 0;
    if (lane == leader) base = atomicAdd(ctr + (isLong ? kCtrShadowCount : kCtrShadowShort), __popc(peers));
    base = __shfl_sync(active, base, leader) + __popc(peers & ((1u << lane) - 1u));
#else
    const uint base = atomicAdd(ctr + (isLong ? kCtrShadowCount : kCtrShadowShort), 1u);
#endif
    return isLong ? base : capacity - 1u - base;
}

// What HandleHit does with a vertex's NEE result once visibility is known (PathTracer.hlsli:725-746): if any half of the packed (radiance, specAvg) is positive,
// AccumulatePathRadiance.  REALTIME (FILL pass): attenuated by 1 / sub-sample count, with the specular average chosen by the sign bits of r.x (shadeHit); reference mode:
// `slot` is the path's home index h.  The shadow kernel applies a single sample's record with it, k_nee_resolve the sum of a block.
template <bool REALTIME>
PT_DEVICE void accumulateNeeRadiance(const LaunchParams& p, uint slot, uint2 r)
{
    const float rx = f16tof32(r.x & 0x7FFFu), ry = f16tof32((r.x >> 16) & 0x7FFFu), rz = f16tof32(r.y), rw = f16tof32(r.y >> 16);
    if (rx > 0 || ry > 0 || rz > 0 || rw > 0)
    {
        if constexpr (REALTIME)
        {
            uint4 s2 = p.wf.s2[slot];
            const float a = p.rt.attenuation;
            const float spec = (r.x & 0x00008000u) ? rw : ((r.x & 0x80000000u) ? (rx + ry + rz) / 3.0f : 0.0f);
            const float lx = f16tof32(s2.z) + rx * a, ly = f16tof32(s2.z >> 16) + ry * a, lz = f16tof32(s2.w) + rz * a, lw = f16tof32(s2.w >> 16) + spec * a;
            s2.z = packHalf2NoClamp(clampf(lx, 0.f, kHalfMax), clampf(ly, 0.f, kHalfMax));
            s2.w = packHalf2NoClamp(clampf(lz, 0.f, kHalfMax), clampf(lw, 0.f, kHalfMax));
            p.wf.s2[slot] = s2;
        }
        else
        {
            uint2 l = p.radiance[slot];
            const float lx = f16tof32(l.x) + rx, ly = f16tof32(l.x >> 16) + ry, lz = f16tof32(l.y) + rz, lw = f16tof32(l.y >> 16);
            l.x = packHalf2NoClamp(clampf(lx, 0.f, kHalfMax), clampf(ly, 0.f, kHalfMax));
            l.y = packHalf2NoClamp(clampf(lz, 0.f, kHalfMax), clampf(lw, 0.f, kHalfMax));
            p.radiance[slot] = l;
        }
    }
}

// k_nee_resolve's body for the block at `block`: the visible samples summed in sample order as NEEResult::AccumulateRadiance does - each fp32 term added to the fp32 value
// of the running fp16 sum, which is rounded back to fp16 after every sample (PathTracerNEE.hlsli:277-346) - then applied once, as the shadow kernel applies one record
template <bool REALTIME>
PT_DEVICE void resolveNeeBlock(const LaunchParams& p, const uint4* block)
{
    const uint4 h = block[0];
    uint2 sum = make_uint2(0u, 0u);
    for (uint j = 0; j <= kNeeMaxFullSamples; j++)
    {
        const uint bit = j < 32 ? (h.z >> j) & 1u : (h.w >> (j - 32)) & 1u;
        if (!bit) continue;
        const uint4 s = block[1 + j];
        sum.x = packHalf2Clamp(f16tof32(sum.x) + __uint_as_float(s.x), f16tof32(sum.x >> 16) + __uint_as_float(s.y));
        sum.y = packHalf2Clamp(f16tof32(sum.y) + __uint_as_float(s.z), f16tof32(sum.y >> 16) + __uint_as_float(s.w));
    }
    sum.x |= h.y;
    accumulateNeeRadiance<REALTIME>(p, h.x, sum);
}

// every lane of the warp calls this; `emit` lanes get the index of their shadow record
PT_DEVICE uint appendShadowRecord(const LaunchParams& p, uint* ctr, bool emit, float tMax)
{
    const uint lane = threadIdx.x & 31u, lt = (1u << lane) - 1u;
    const bool isLong = emit && tMax > p.shadowLongRayT;
    const uint longPeers = __ballot_sync(0xFFFFFFFFu, isLong), shortPeers = __ballot_sync(0xFFFFFFFFu, emit && !isLong);
    uint bl = 0, bs = 0;
    if (longPeers && lane == __ffs(longPeers) - 1u) bl = atomicAdd(ctr + kCtrShadowCount, __popc(longPeers));
    if (shortPeers && lane == __ffs(shortPeers) - 1u) bs = atomicAdd(ctr + kCtrShadowShort, __popc(shortPeers));
    if (longPeers) bl = __shfl_sync(0xFFFFFFFFu, bl, __ffs(longPeers) - 1);
    if (shortPeers) bs = __shfl_sync(0xFFFFFFFFu, bs, __ffs(shortPeers) - 1);
    return isLong ? bl + __popc(longPeers & lt) : p.wf.capacity - 1u - (bs + __popc(shortPeers & lt));
}

// ---- stable-plane addressing (GenericTS, Utils.hlsli:320-362; StablePlanes.hlsli:120-140): host+device so that the denoiser interface's pixel bodies also build for the host ----
constexpr uint kInvalidBranchID = 0xFFFFFFFFu;
#ifdef __CUDA_ARCH__
PT_HD uint vertexIndexFromBranchID(uint id) { return (31u - __clz(id)) / 2u + 1u; }       // firstbithigh(id)/2 + 1
#else
PT_HD uint vertexIndexFromBranchID(uint id) { return (31u - uint(__builtin_clz(id))) / 2u + 1u; }
#endif
PT_HD uint morton16(uint x, uint y)
{
    uint t = (x & 0xffu) | ((y & 0xffu) << 16);
    t = (t ^ (t << 4)) & 0x0f0f0f0fu; t = (t ^ (t << 2)) & 0x33333333u; t = (t ^ (t << 1)) & 0x55555555u;
    return ((t >> 15) | t) & 0xffffu;
}
PT_HD uint planeAddress(const RealtimeParams& rt, uint id, uint plane)
{
    const uint px = id >> 16, py = id & 0xFFFFu, xi = px & 7u, yi = py & 7u;
    return (px - xi) * 8u + (py - yi) * rt.lineStride + morton16(xi, yi) + plane * rt.planeStride;
}
PT_HD uint& headerWord(const LaunchParams& p, uint id, uint layer)
{
    return p.rt.header[(size_t(layer) * p.c.imageHeight + (id & 0xFFFFu)) * p.c.imageWidth + (id >> 16)];
}
PT_HD size_t pixelOffset(const LaunchParams& p, uint id) { return size_t(id & 0xFFFFu) * p.c.imageWidth + (id >> 16); }

// ---- packed path-state accessors (PathState.hlsli:125-200) ------------------------------------------------------------------
enum : uint {
    kPFActive = 1u << 0, kPFHit = 1u << 1, kPFTransmission = 1u << 2, kPFSpecular = 1u << 3, kPFDelta = 1u << 4,
    kPFInsideDielectric = 1u << 5, kPFTerminateAtNextBounce = 1u << 6, kPFEnableThreadReorder = 1u << 9, kPFDeltaOnlyPath = 1u << 12,
    // realtime mode (PathState.hlsli:58-64); flag bits 14-15 hold the stable plane index
    kPFStablePlaneOnPlane = 1u << 16, kPFStablePlaneOnBranch = 1u << 17, kPFStablePlaneBaseScatterDiff = 1u << 18, kPFExportSpecHitTQueued = 1u << 19,
    kPFStablePlaneOnDominantBranch = 1u << 20
};
constexpr int kModeReference = 0, kModeBuildStablePlanes = 1, kModeFillStablePlanes = 2;      // PATH_TRACER_MODE (Config.h:56-59)
constexpr uint kVertexIndexBits = 10, kVertexIndexMask = (1u << kVertexIndexBits) - 1u;
constexpr uint kStablePlaneIndexShift = 14 + kVertexIndexBits, kStablePlaneIndexMask = 3u << kStablePlaneIndexShift;

// Path state is written once and read once per wavefront iteration: with PT_STREAM_STATE the accesses carry the evict-first hint so that they
// do not displace BVH and scene data in L2.
#ifndef PT_STREAM_STATE
#define PT_STREAM_STATE 0
#endif
#if PT_STREAM_STATE
PT_DEVICE uint4 ldState(const uint4* p) { return __ldcs(p); }
PT_DEVICE void stState(uint4* p, uint4 v) { __stcs(p, v); }
#else
PT_DEVICE uint4 ldState(const uint4* p) { return *p; }
PT_DEVICE void stState(uint4* p, uint4 v) { *p = v; }
#endif

struct PathRegs             // one path's state in registers
{
    float3 origin; uint id;
    float3 dir; float sceneLength;
    uint thpXY, thpZ;       // fp16 pairs
    uint lXY, lZW;
    uint interior0, interior1, packedCounters, rayCone;
    uint pack0, pack1, flagsAndVertexIndex, sampleIndex;

    PT_DEVICE void load(const WavefrontBuffers& w, uint slot, bool needRay)
    {
        if (needRay)
        {
            const uint4 a = ldState(w.s0 + slot), b = ldState(w.s1 + slot);
            origin = mk3(__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z)); id = a.w;
            dir = mk3(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z)); sceneLength = __uint_as_float(b.w);
        }
        const uint4 c = ldState(w.s2 + slot), d = ldState(w.s3 + slot), e = ldState(w.s4 + slot);
        thpXY = c.x; thpZ = c.y; lXY = c.z; lZW = c.w;
        interior0 = d.x; interior1 = d.y; packedCounters = d.z; rayCone = d.w;
        pack0 = e.x; pack1 = e.y; flagsAndVertexIndex = e.z; sampleIndex = e.w;
    }
    PT_DEVICE void store(const WavefrontBuffers& w, uint slot) const
    {
        stState(w.s0 + slot, make_uint4(__float_as_uint(origin.x), __float_as_uint(origin.y), __float_as_uint(origin.z), id));
        stState(w.s1 + slot, make_uint4(__float_as_uint(dir.x), __float_as_uint(dir.y), __float_as_uint(dir.z), __float_as_uint(sceneLength)));
        stState(w.s2 + slot, make_uint4(thpXY, thpZ, lXY, lZW));
        stState(w.s3 + slot, make_uint4(interior0, interior1, packedCounters, rayCone));
        stState(w.s4 + slot, make_uint4(pack0, pack1, flagsAndVertexIndex, sampleIndex));
    }
    // a path that ends at this vertex is only read again for its radiance (shadow kernel, commit): 16 of the 80 bytes
    PT_DEVICE void storeRadianceOnly(const WavefrontBuffers& w, uint slot) const { stState(w.s2 + slot, make_uint4(thpXY, thpZ, lXY, lZW)); }
    // reference mode: ray r of a state set; returns the path's home index h, whose radiance L is loaded from `radiance`
    PT_DEVICE uint loadRay(const StateSet& st, uint r, const uint2* radiance)
    {
        const uint4 a = ldState(st.s0 + r), b = ldState(st.s1 + r), c = ldState(st.s2 + r), d = ldState(st.s3 + r), e = ldState(st.s4 + r);
        origin = mk3(__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z)); id = a.w;
        dir = mk3(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z)); sceneLength = __uint_as_float(b.w & 0x7FFFFFFFu);
        thpXY = c.x; thpZ = c.y;
        interior0 = d.x; interior1 = d.y; packedCounters = d.z; rayCone = d.w;
        pack0 = e.x; pack1 = e.y; flagsAndVertexIndex = e.z; sampleIndex = e.w;
        const uint2 l = radiance[c.z]; lXY = l.x; lZW = l.y;
        return c.z;
    }
    PT_DEVICE void storeRay(const StateSet& st, uint r, uint h) const
    {
        const uint terminate = hasFlag(kPFTerminateAtNextBounce) ? 0x80000000u : 0u;
        stState(st.s0 + r, make_uint4(__float_as_uint(origin.x), __float_as_uint(origin.y), __float_as_uint(origin.z), id));
        stState(st.s1 + r, make_uint4(__float_as_uint(dir.x), __float_as_uint(dir.y), __float_as_uint(dir.z), __float_as_uint(sceneLength) | terminate));
        stState(st.s2 + r, make_uint4(thpXY, thpZ, h, 0u));
        stState(st.s3 + r, make_uint4(interior0, interior1, packedCounters, rayCone));
        stState(st.s4 + r, make_uint4(pack0, pack1, flagsAndVertexIndex, sampleIndex));
    }
    PT_DEVICE void storeRadiance(uint2* radiance, uint h) const { radiance[h] = make_uint2(lXY, lZW); }
    PT_DEVICE float3 thp() const { return mk3(f16tof32(thpXY), f16tof32(thpXY >> 16), f16tof32(thpZ)); }
    PT_DEVICE void setThp(float3 t) { thpXY = packHalf2NoClamp(clampf(t.x, 0.f, kHalfMax), clampf(t.y, 0.f, kHalfMax)); thpZ = packHalf2NoClamp(clampf(t.z, 0.f, kHalfMax), 0.f); }
    PT_DEVICE float4 L() const { return make_float4(f16tof32(lXY), f16tof32(lXY >> 16), f16tof32(lZW), f16tof32(lZW >> 16)); }
    PT_DEVICE void setL(float4 l) { lXY = packHalf2NoClamp(clampf(l.x, 0.f, kHalfMax), clampf(l.y, 0.f, kHalfMax)); lZW = packHalf2NoClamp(clampf(l.z, 0.f, kHalfMax), clampf(l.w, 0.f, kHalfMax)); }
    PT_DEVICE void addRadiance(float3 r) { float4 l = L(); setL(make_float4(l.x + r.x, l.y + r.y, l.z + r.z, l.w)); }    // AccumulatePathRadiance, PathTracer.hlsli:139-143
    PT_DEVICE float fireflyK() const { return f16tof32(pack0 >> 16); }
    PT_DEVICE float bsdfScatterPdf() const { return f16tof32(pack0); }
    PT_DEVICE void setFireflyK_BsdfPdf(float k, float pdf) { pack0 = (f32tof16(clampf(k, 0.f, kHalfMax)) << 16) | f32tof16(clampf(pdf, 0.f, kHalfMax)); }
    PT_DEVICE uint misInfo() const { return pack1 >> 16; }
    PT_DEVICE float ruRuCorrection() const { return f16tof32(pack1); }
    PT_DEVICE void setMisInfo_RuRu(uint mis, float c) { pack1 = (mis << 16) | f32tof16(clampf(c, 0.f, kHalfMax)); }
    PT_DEVICE bool hasFlag(uint f) const { return (flagsAndVertexIndex & (f << kVertexIndexBits)) != 0; }
    PT_DEVICE void setFlag(uint f, bool v) { const uint bit = f << kVertexIndexBits; flagsAndVertexIndex = v ? (flagsAndVertexIndex | bit) : (flagsAndVertexIndex & ~bit); }
    PT_DEVICE uint vertexIndex() const { return flagsAndVertexIndex & kVertexIndexMask; }
    PT_DEVICE uint counter(uint type) const { return (packedCounters >> (type << 3)) & 0xff; }
    PT_DEVICE void incrementCounter(uint type) { packedCounters += 1u << (type << 3); }
    PT_DEVICE void setCounter(uint type, uint v) { const uint shift = type << 3; packedCounters = (packedCounters & ~(0xffu << shift)) | ((v & 0xffu) << shift); }
    PT_DEVICE void setVertexIndex(uint v) { flagsAndVertexIndex = (flagsAndVertexIndex & ~kVertexIndexMask) | v; }
    PT_DEVICE uint stablePlaneIndex() const { return (flagsAndVertexIndex & kStablePlaneIndexMask) >> kStablePlaneIndexShift; }
    PT_DEVICE void setStablePlaneIndex(uint i) { flagsAndVertexIndex = (flagsAndVertexIndex & ~kStablePlaneIndexMask) | (i << kStablePlaneIndexShift); }
    // realtime mode: every path of a launch has the launch's sample index, and the word carries PathState::stableBranchID as in the reference payload;
    // in the BUILD pass lXY/lZW hold imageXformPacked and pack0 the motion-vector scene length (PathState.hlsli:91-92, :151-154)
    PT_DEVICE uint& stableBranchID() { return sampleIndex; }
    PT_DEVICE float coneWidth() const { return f16tof32(rayCone >> 16); }
    PT_DEVICE float coneSpread() const { return f16tof32(rayCone); }
    PT_DEVICE void setCone(float width, float spread) { rayCone = (f32tof16(width) << 16) | f32tof16(spread); }
};
constexpr uint kCtrDiffuseBounces = 0, kCtrRejectedHits = 1, kCtrBouncesFromStablePlane = 2;

// Bridge::computeCameraRay + ComputeRayThinlens (BridgeDonut:543-564, PathTracerHelpers.hlsli:126-153): camera ray of pixel `id` for sample `sampleIndex`
#ifdef PT_HOST_EMU     // tests/emu/shade_host_emu.cu (test infrastructure): the camera and the motion-vector projection are the golden vectors' stub bridge's closed forms
__host__ __device__ void emuCameraRay(uint id, float3& origin, float3& dir);
__host__ __device__ float3 emuMotionVector(float3 posW, float3 prevPosW);
#endif
PT_HD void computeCameraRay(const RtxptPathTracerConstants& c, uint id, uint sampleIndex, float3& origin, float3& dir)
{
#ifdef PT_HOST_EMU
    emuCameraRay(id, origin, dir); return;
#endif
    const RtxptCameraData& cam = c.camera;
    const uint px = id >> 16, py = id & 0xFFFF;
    UniformSeq sg = UniformSeq::make(vertexBaseHash(id, 0), sampleIndex, 0u);
    const float r0 = sg.next(), r1 = sg.next(), d0 = sg.next(), d1 = sg.next();
    const float jx = cam.Jitter[0] + (r0 - 0.5f) * c.perPixelJitterAAScale, jy = cam.Jitter[1] + (r1 - 0.5f) * c.perPixelJitterAAScale;
    const float sx = (float(px) + 0.5f + (-jx)) / float(cam.ViewportSize[0]), sy = (float(py) + 0.5f + jy) / float(cam.ViewportSize[1]);
    const float ndcx = 2.f * sx - 1.f, ndcy = -2.f * sy + 1.f;
    const float3 U = mk3(cam.CameraU[0], cam.CameraU[1], cam.CameraU[2]), V = mk3(cam.CameraV[0], cam.CameraV[1], cam.CameraV[2]), W = mk3(cam.CameraW[0], cam.CameraW[1], cam.CameraW[2]);
    origin = mk3(cam.PosW[0], cam.PosW[1], cam.PosW[2]);
    dir = ndcx * U + ndcy * V + W;
    const float2 ap = sampleDiskPolar(d0, d1);
    const float3 target = origin + dir;
    origin = origin + cam.ApertureRadius * (ap.x * norm3(U) + ap.y * norm3(V));
    dir = norm3(target - origin);
    const float invCos = 1.f / dot3(norm3(W), dir);
    origin = origin + dir * (cam.NearZ * invCos);
}

// guide export (Bridge::ExportSurface / ExportNonSurface, BridgeDonut:1105-1146): only the last sub-sample of a launch writes, as the
// reference's sequential sub-sample dispatches leave the last one in the buffers
PT_DEVICE uint packR11G11B10(float3 rgb)        // Utils/Packing.hlsli:175-184
{
    const float top = __uint_as_float(0x477C0000u);
    const uint r = ((f32tof16(fminf(rgb.x, top)) + 8u) >> 4) & 0x000007FFu;
    const uint g = ((f32tof16(fminf(rgb.y, top)) + 8u) << 7) & 0x003FF800u;
    const uint b = ((f32tof16(fminf(rgb.z, top)) + 16u) << 17) & 0xFFC00000u;
    return r | g | b;
}
PT_DEVICE void exportGuide(const LaunchParams& p, uint id, float3 worldPos, uint packedThroughput)
{
    const float* M = p.worldToClip;
    const float z = worldPos.x * M[2] + worldPos.y * M[6] + worldPos.z * M[10] + M[14], w = worldPos.x * M[3] + worldPos.y * M[7] + worldPos.z * M[11] + M[15];
    const size_t o = size_t(id & 0xFFFF) * p.c.imageWidth + (id >> 16);
    p.depth[o] = z / w; p.throughput[o] = packedThroughput; p.motionVectors[o] = make_uint2(0u, 0u);
}

PT_DEVICE bool hasFinishedSurfaceBounces(const RtxptPathTracerConstants& c, uint vertexIndex, uint diffuseBounces)   // PathTracer.hlsli:40-45
{
    if (c.bounceCount < vertexIndex) return true;
    return diffuseBounces > c.diffuseBounceCount;
}

} // namespace pt
