// api.cu — implementation of the C ABI declared in include/rtxpt_b200.h: context, scene upload (tables, textures, BVH, lights),
// constants, the wavefront launch sequence, read-back and the inspection hooks.
// Host orchestration mirrors the slice of Sample::Render that surrounds the dispatch (Rtxpt/Sample.cpp:2008-2186): acceleration
// structure build, MaterialsBaker::Update, UpdateLighting, constant-buffer write, PathTrace, AccumulationPass.
// There is no CPU rendering fallback anywhere in this library: without a CUDA device every entry point fails with RTXPT_ERR_NO_DEVICE.
#include "kernels.h"
#include "debug_views.cuh"
#include "denoiser_iface.cuh"
#include "opacity_masks.h"
#include "reblur_host.h"
#include "neeat_host.h"
#include "envbake.cuh"
#include "refit.cuh"
#include "bvh_build.cuh"
#include "scan.cuh"
#include "tonemap.cuh"
#include "skinning.cuh"
#include "lights_bake.h"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <memory>
#include <string>
#include <utility>
#include <vector>

using namespace pt;
namespace rtxpt_host { void decodeBlocksToRgba8(uint32_t format, const uint8_t* blocks, uint32_t w, uint32_t h, std::vector<uint8_t>& rgba); }      // dds.cpp

static_assert(sizeof(RtxptGeometryData) == 64, "GeometryData layout");
static_assert(sizeof(RtxptInstanceData) == 112, "InstanceData layout");
static_assert(sizeof(RtxptSubInstanceData) == 32, "SubInstanceData layout");
static_assert(sizeof(RtxptMaterialData) == 128, "PTMaterialData layout");
static_assert(sizeof(RtxptCameraData) == 112, "PathTracerCameraData layout");
static_assert(sizeof(LightInfo) == 32 && sizeof(BakedLight) == 32, "PolymorphicLightInfo layout");
static_assert(sizeof(Bvh8Node) == 80 && sizeof(Bvh8Tri) == 48, "CWBVH8 layout");
static_assert(sizeof(RtxptStablePlane) == 80, "StablePlane layout (StablePlanes.hlsli:48-80)");
static_assert(sizeof(LaunchParams) <= 4000, "kernel parameter block");

static thread_local std::string g_lastError;
static int fail(int code, const char* fmt, ...)
{
    char buf[1024]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_lastError = buf; return code;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(e_ == cudaErrorMemoryAllocation ? RTXPT_ERR_OUT_OF_MEMORY : RTXPT_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

// Every CUDA resource the library holds belongs to one of the two owner types below, so that an early return (CU) or a destroyed context frees
// whatever was made so far.  g_liveResources counts what they hold across the process (rtxpt_b200_debug_live_resources).
static std::atomic<uint64_t> g_liveResources{ 0 };

template <typename T> struct DeviceArray
{
    T* ptr = nullptr; size_t count = 0;
    DeviceArray() = default; DeviceArray(const DeviceArray&) = delete; DeviceArray& operator=(const DeviceArray&) = delete;
    DeviceArray(DeviceArray&& o) noexcept : ptr(std::exchange(o.ptr, nullptr)), count(std::exchange(o.count, 0)) {}
    DeviceArray& operator=(DeviceArray&& o) noexcept { if (this != &o) { reset(); ptr = std::exchange(o.ptr, nullptr); count = std::exchange(o.count, 0); } return *this; }
    ~DeviceArray() { reset(); }
    cudaError_t alloc(size_t n) { reset(); if (n == 0) return cudaSuccess; cudaError_t e = cudaMalloc(&ptr, n * sizeof(T)); if (e != cudaSuccess) { ptr = nullptr; return e; } g_liveResources++; count = n; return cudaSuccess; }
    cudaError_t upload(const T* src, size_t n, cudaStream_t s) { cudaError_t e = alloc(n); if (e != cudaSuccess || n == 0) return e; return cudaMemcpyAsync(ptr, src, n * sizeof(T), cudaMemcpyHostToDevice, s); }
    cudaError_t fill(int byte, cudaStream_t s) const { return cudaMemsetAsync(ptr, byte, count * sizeof(T), s); }
private:
    void reset() { if (ptr) { cudaFree(ptr); g_liveResources--; } ptr = nullptr; count = 0; }
};

// one stream, event, texture object, mipmapped array or pinned host block, destroyed by Destroy; reads as the raw handle
template <typename T, auto Destroy> struct Owned
{
    Owned() = default; Owned(const Owned&) = delete; Owned& operator=(const Owned&) = delete;
    Owned(Owned&& o) noexcept : h(std::exchange(o.h, T{})) {}
    Owned& operator=(Owned&& o) noexcept { if (this != &o) { reset(); h = std::exchange(o.h, T{}); } return *this; }
    ~Owned() { reset(); }
    operator T() const { return h; }
    // make(&handle, args...): a CUDA creation call; replaces what was held before
    template <typename F, typename... A> cudaError_t create(F make, A... args) { reset(); cudaError_t e = make(&h, args...); if (e != cudaSuccess) h = T{}; else if (h) g_liveResources++; return e; }
private:
    T h{};
    void reset() { if (h) { Destroy(h); g_liveResources--; } h = T{}; }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;

// members are destroyed in reverse order: the texture object before its array
struct DeviceTexture
{
    Owned<cudaMipmappedArray_t, cudaFreeMipmappedArray> array; Owned<cudaTextureObject_t, cudaDestroyTextureObject> object;
    Owned<cudaTextureObject_t, cudaDestroyTextureObject> pointObject;         // the same arrays, point-filtered: stochastic texture filtering fetches one texel
};

struct rtxpt_ctx
{
    RtxptConfig cfg{};
    int device = 0;
    // streams and events come before the buffers, so that they outlive them when the context is destroyed
    Stream stream;
    // pipeline lanes: the sub-samples of one launch are split into independent wavefronts, each on its own pair of streams, so that the latency-bound tail of every
    // persistent kernel of one lane (its last, longest rays) is filled by the CTAs of the other lanes.  Lane 0's first stream is the caller's (its `s` stays empty).
    static const int kMaxLanes = 8;
    struct Lane { Stream s, s2; Event evShadeDone, evShadowDone, evCommitted; } lanes[kMaxLanes];
    Event evFork, evStart, evStop;
    Event evDnStart, evDnStop;          // around the last rtxpt_b200_denoise_realtime
    std::vector<Event> evPool;          // RTXPT_CFG_TIME_KERNELS: (begin,end) pairs per kernel
    Event evCallerJoin;                 // joins lastCallerStream into `stream` (joinCallerStream)
    GridConfig grid;
    int maxSmemOptin = 0;
    // scene
    bool haveScene = false, haveConstants = false, lightsDirty = true; uint64_t lightVersion = 0;       // bumped by every re-bake of the light list (uploadLights)
    size_t l2PersistBytes = 0, l2WindowMax = 0;
    // measurement knobs, read from the environment once at creation (RTXPT_* variables; the defaults measured fastest on an H100 SXM at a 400 W power limit, bench.py workload: see the launch configuration)
    struct Tuning { int refillThreshold = 24, waitFlushLanes = 8, traceCtas = 4, shadeCtas = 4, smemNodes = 0, lanes = 1, shadowLpt = 1; } tune; float sceneDiagonal = 0;
    bool overlapShadow = true; uint32_t lastLanes = 1, lastSubSamplesPerLaunch = 1;
    DeviceArray<RtxptInstanceData> dInstances; DeviceArray<RtxptGeometryData> dGeometries; DeviceArray<RtxptSubInstanceData> dSubInstances;
    DeviceArray<RtxptMaterialData> dMaterials; DeviceArray<uint8_t> dSubInstanceClass;
    std::vector<DeviceArray<uint8_t>> bufferAllocs; DeviceArray<const uint8_t*> dBufferTable;
    std::vector<DeviceTexture> textures; DeviceArray<cudaTextureObject_t> dTextureTable;
    DeviceArray<cudaTextureObject_t> dPointTextureTable; DeviceArray<uint4> dTextureDims;     // stochastic texture filtering: point-filtered objects, width / height / levels
    RtxptStochasticTextureFiltering stf{};                                                  // rtxpt_b200_set_texture_filtering (off)
    RtxptDebugView debugView{}; DeviceArray<uint2> debugViz;                                 // rtxpt_b200_set_debug_view (disabled); RGBA16F, allocated by the first call that draws
    DeviceTexture envCube; uint32_t envFaceSize = 0, envMipLevels = 0;
    // rtxpt_b200_update_env_map: the bake's linear MIP chain and the importance map's, grown to the largest cube baked and never shrunk; the source of the last update, kept so
    // that the next update can re-bake from it; event times of the last update (bake, importance map, copy into the cube, readback + light bake + upload)
    DeviceArray<float> envBakeScratch, envImportanceScratch, envSource; uint32_t envSourceType = 0, envSourceWidth = 0, envSourceHeight = 0;
    Event evEnv[5]; float envUpdateMs[4] = {};
    DeviceArray<uint4> dBvhNodes; DeviceArray<float4> dBvhTris; DeviceArray<uint4> dTriInfo, dTriShade, dOpacityMasks;
    uint32_t opacityMaskTriangles = 0; uint64_t opacityMaskStates[3] = { 0, 0, 0 }; float opacityMaskBakeSeconds = 0;
    std::vector<RtxptInstanceData> hInstances; std::vector<uint32_t> bvhLevelStart; DeviceArray<float> dNodeBox;      // rigid-instance animation (refit.cuh)
    // skinned meshes (skinning.cuh): where each (instance, geometry)'s triangles start in gid order, its index range on the device, and the registered bind poses
    std::vector<RtxptGeometryData> hGeometries; std::vector<uint32_t> firstGidOfSubInstance; std::vector<const uint8_t*> hBufferTable; std::vector<uint32_t> maxVertexOfSubInstance;      // largest vertex index each sub-instance's triangles name (skin registration validates against it)
    // last frame's object-space corners of geometries with a previous-position stream (scene_device.cuh: prevPosBase / triPrevPos)
    std::vector<uint32_t> hPrevPosBase; DeviceArray<uint32_t> dPrevPosBase; DeviceArray<float> dTriPrevPos; size_t prevPosTriangles = 0;
    struct Skin { uint32_t numVertices = 0, numTriangles = 0, firstGid = 0, flags = 0, numJoints = 0, maxJoint = 0, prevPosFirst = 0; const uint32_t* dIndices = nullptr;
                  DeviceArray<float> positions, weights, outPositions, jointMatrices; DeviceArray<uint32_t> normals, tangents, outNormals, outTangents; DeviceArray<unsigned short> jointIndices; };
    std::vector<std::unique_ptr<Skin>> skins;
    uint32_t bvhNodeCount = 0, bvhTriCount = 0; float bvhBuildSeconds = 0;
    float bvhRootBox[6] = {};           // exact box of the root as last built (the host build's scene bounds, or the device rebuild's root box): the SAH statistics' reference area
    // device rebuild (bvh_build.cuh): scratch grown to the largest scene rebuilt, never shrunk; the new tree is built into `nodes` / `outTris` and swapped in on success
    struct BvhScratch { DeviceArray<float4> tris, outTris; DeviceArray<uint4> nodes; DeviceArray<float> nodeBox, box2; DeviceArray<unsigned long long> keys[2], hist, flags, scanBlocks, misc;
                        DeviceArray<uint32_t> vals[2], count2, clusters[2], nn, nodeRoot, cenBounds; DeviceArray<uint2> child2; } bvhScratch;
    Event evBvhStart, evBvhStop;
    std::vector<RtxptSubInstanceData> hSubInstances; uint32_t materialCount = 0;
    LightBakeState lightState;
    DeviceArray<LightInfo> dLights; DeviceArray<uint32_t> dProxyCounters, dProxyIndices, dEnvLookup; DeviceArray<uint4> dLightsEx;
    // wavefront
    DeviceArray<uint4> s0, s1, s2, s3, s4; DeviceArray<float4> hits; DeviceArray<uint32_t> rayQueue[2], shadeQueue;
    DeviceArray<uint4> t0, t1, t2, t3, t4; DeviceArray<uint2> radiance;        // reference mode: second path-state set, radiance per home index (wavefront.cuh)
    DeviceArray<float4> shadowOriginTMax, shadowDirPath; DeviceArray<uint2> shadowRadiance;
    // NEEFullSamples > 1: shadow records of every light sample and the NEE blocks (wavefront.cuh), allocated by the first trace that needs them (ensureNeeSamples)
    struct NeeSamples { DeviceArray<float4> originTMax, dirPath; DeviceArray<uint2> sample; DeviceArray<uint4> blocks; } neeSamples;
    DeviceArray<uint32_t> counters; DeviceArray<uint32_t> pixelOfSlot, allPixelTable;
    uint32_t paddedPixelsPerRank = 0;
    uint32_t capacity = 0, pixelCount = 0, tableWidth = 0, tableHeight = 0;
    // render targets
    DeviceArray<uint2> outputColor; DeviceArray<float4> accumulated; DeviceArray<float> depth; DeviceArray<uint2> motionVectors; DeviceArray<uint32_t> throughput; float worldToClip[16] = {}; bool haveView = false;
    uint32_t accumulatedSamples = 0;
    RtxptPathTracerConstants consts{};
    // realtime mode (stable planes): allocated on the first set_realtime for the current image size
    DeviceArray<RtxptStablePlane> stablePlanes; DeviceArray<uint32_t> stablePlanesHeader; DeviceArray<uint2> stableRadiance; DeviceArray<float> specularHitT;
    RtxptRealtimeConstants realtime{}; bool haveRealtime = false; uint32_t realtimeWidth = 0, realtimeHeight = 0;
    // denoiser interface: NRD's inputs for one plane at a time (allocated by the first prepare_inputs call)
    DeviceArray<float> dnViewZ; DeviceArray<uint2> dnMotion, dnDiff, dnSpec; DeviceArray<uint32_t> dnNormalRoughness; DeviceArray<uint8_t> dnDisocclusionMix, dnHistoryClampRelax;
    uint32_t denoiserWidth = 0, denoiserHeight = 0;
    uint32_t realtimeFrameWidth = 0, realtimeFrameHeight = 0;         // image size of the last rtxpt_b200_path_trace_realtime (0: none yet)
    // DLSS-RR inputs (rtxpt_b200_dlss_rr_prepare_inputs): R11G11B10 diffuse / specular albedo, RGBA16F normals + roughness, RG16F specular motion vectors; allocated by the first call
    DeviceArray<uint32_t> rrDiffAlbedo, rrSpecAlbedo, rrSpecMotionVectors; DeviceArray<uint2> rrNormalsRoughness; uint32_t rrWidth = 0, rrHeight = 0;
    DeviceArray<float> dnScratchFloat;          // ping-pong partner of the specular hit distance guide (DenoiseSpecHitT)
    // ReBLUR: one permanent pool per stable plane (RTXPT keeps one NRD instance per plane, Sample.cpp:2560-2618), one transient pool and one pair of outputs shared by all
    struct ReblurHistory
    {
        DeviceArray<float> prevViewZ; DeviceArray<uint32_t> prevNormalRoughness; DeviceArray<uint16_t> prevInternalData, diffFast, specFast, tracking[2], diffLuma[2], specLuma[2];
        DeviceArray<uint2> diffHistory, specHistory; bool valid = false; uint32_t pingPong = 0;
    } reblur[RTXPT_STABLE_PLANE_COUNT];
    RtxptReblurSettings reblurSettings = rb::defaultSettings();                                 // rtxpt_b200_set_reblur_settings; every plane's instance denoises with them
    DeviceArray<uint8_t> rbTiles; DeviceArray<uint2> rbTmp1Diff, rbTmp1Spec, rbTmp2Diff, rbTmp2Spec, rbOutDiff, rbOutSpec; DeviceArray<uint16_t> rbTrackingT, rbDiffFastT, rbSpecFastT; DeviceArray<uchar2> rbData1; DeviceArray<uint32_t> rbData2;
    uint32_t reblurWidth = 0, reblurHeight = 0;
    // NEE-AT temporal feedback (consts.NEEType == 2 && consts.NEEATFeedback): LightsBaker's frame state, reservoirs, tile samplers and the per-frame global proxy table
    struct Neeat
    {
        neeat::HostState host; neeat::Params params{}; bool allocated = false, frameBegun = false, frameEnded = false; uint32_t lightCount = 0;      // begun: update_begin ran, update_end pending; ended: both ran
        DeviceArray<float> fbWeight, scratchWeight, blendedWeight, historyDepth, lightWeights; DeviceArray<uint32_t> fbCandidate, scratchCandidate, blendedCandidate, local, counters,
            proxyCounters, proxyOffsets, proxyIndices, samplingProxyCount, scanBlockSums, rrFix; DeviceArray<uint4> shadowFeedback;
        DeviceArray<float> weights[2], weightGroupSums, weightsSum; uint32_t weightPingPong = 0;      // boosted weights: this frame / last frame
        // dynamic light lists: the list last frame's feedback was indexed by, and this frame's past <-> current index tables (NULL pointers in params while the list stands still)
        LightListSnapshot snap; uint64_t snapVersion = 0; bool remapActive = false; uint32_t lightCapacity = 0; DeviceArray<uint32_t> pastToCurrent, currentToPast; std::vector<uint32_t> hPastToCurrent, hCurrentToPast;
    } na;
    DeviceArray<double> tmPartials; DeviceArray<float> tmAvgLuminance; DeviceArray<uint32_t> ldrColor; bool toneMapped = false;      // tone mapping (tonemap.cuh)
    bool denoiseTimed = false;
    // stats
    Owned<uint32_t*, cudaFreeHost> hCounters;          // pinned
    std::vector<int> evKind; size_t evUsed = 0;
    uint32_t lastIterations = 0, lastSubSamples = 0; uint64_t lastLaunches = 0;
    bool statsPending = false;
    // the caller's stream that last received work through this context (null: everything went to `stream`); host reads join it first
    cudaStream_t lastCallerStream = nullptr;
};

static const uint32_t kCounterWords = (kMaxWavefrontIterations + 2) * kCountersPerIter;

// Work goes to the caller's stream when one is passed, otherwise to the context's own (non-blocking) stream; there is no implicit ordering between the two.  Every entry point
// that hands results to the host (readback, synchronize, get_stats, the NEE-AT / tone-map getters) therefore first makes the context stream wait for what the caller's stream
// has been given: an event recorded there, waited on here.  One caller stream at a time (calls on a context are serialised by the caller, include/rtxpt_b200.h).
static cudaStream_t pickStream(rtxpt_ctx* c, void* cudaStream)
{
    if (!cudaStream || (cudaStream_t)cudaStream == c->stream) return c->stream;
    c->lastCallerStream = (cudaStream_t)cudaStream;
    return c->lastCallerStream;
}
static cudaError_t joinCallerStream(rtxpt_ctx* c)
{
    if (!c->lastCallerStream) return cudaSuccess;
    cudaError_t e;
    if (!c->evCallerJoin && (e = c->evCallerJoin.create(cudaEventCreateWithFlags, cudaEventDisableTiming)) != cudaSuccess) return e;
    if ((e = cudaEventRecord(c->evCallerJoin, c->lastCallerStream)) != cudaSuccess) return e;
    return cudaStreamWaitEvent(c->stream, c->evCallerJoin, 0);
}
static cudaError_t syncContext(rtxpt_ctx* c) { cudaError_t e = joinCallerStream(c); return e != cudaSuccess ? e : cudaStreamSynchronize(c->stream); }

extern "C" RTXPT_API const char* rtxpt_b200_last_error(void) { return g_lastError.c_str(); }

static void releaseScene(rtxpt_ctx* c)
{
    c->skins.clear(); c->bufferAllocs.clear(); c->textures.clear();
    std::exchange(c->envCube, DeviceTexture());        // the old cube is destroyed at the end of the statement, its texture object before its array
    c->haveScene = false;
}

extern "C" RTXPT_API int rtxpt_b200_create(const RtxptConfig* config, rtxpt_ctx** outCtx)
{
    if (!config || !outCtx) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) return fail(RTXPT_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback", cudaGetErrorString(e));
    std::unique_ptr<rtxpt_ctx> c(new rtxpt_ctx());
    c->cfg = *config;
    if (c->cfg.maxSubSamplesPerLaunch == 0) c->cfg.maxSubSamplesPerLaunch = 1;
    if (c->cfg.tileWorld == 0) { c->cfg.tileWorld = 1; c->cfg.tileRank = 0; }
    if (c->cfg.tileSize == 0) c->cfg.tileSize = 64;
    if (c->cfg.tileRank >= c->cfg.tileWorld || (c->cfg.tileSize & (c->cfg.tileSize - 1)) != 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad tile partition");
    if (config->deviceOrdinal >= 0) { if (cudaSetDevice(config->deviceOrdinal) != cudaSuccess) return fail(RTXPT_ERR_NO_DEVICE, "cudaSetDevice(%d) failed", config->deviceOrdinal); }
    cudaGetDevice(&c->device);
    cudaDeviceProp prop; cudaGetDeviceProperties(&prop, c->device);
    c->grid.smCount = prop.multiProcessorCount;
    c->maxSmemOptin = int(prop.sharedMemPerBlockOptin);
    CU(c->stream.create(cudaStreamCreateWithFlags, cudaStreamNonBlocking));
    CU(c->evStart.create(cudaEventCreateWithFlags, cudaEventDefault)); CU(c->evStop.create(cudaEventCreateWithFlags, cudaEventDefault));
    { const char* e = getenv("RTXPT_OVERLAP_SHADOW"); if (e) c->overlapShadow = atoi(e) != 0; }
    auto envInt = [](const char* name, int def, int lo, int hi) { const char* e = getenv(name); return e ? std::min(hi, std::max(lo, atoi(e))) : def; };
    c->tune.refillThreshold = envInt("RTXPT_REFILL_THRESHOLD", 24, 1, 32); c->tune.waitFlushLanes = envInt("RTXPT_WAIT_FLUSH", 8, 1, 33);
    c->tune.traceCtas = envInt("RTXPT_TRACE_CTAS", 4, 2, 4); c->tune.shadeCtas = envInt("RTXPT_SHADE_CTAS", 4, 3, 5); c->tune.smemNodes = envInt("RTXPT_SMEM_NODES", 0, 0, 1 << 20);
    c->tune.shadowLpt = envInt("RTXPT_SHADOW_LPT", 1, 0, 1);
    c->tune.lanes = envInt("RTXPT_LANES", 1, 1, rtxpt_ctx::kMaxLanes);          // H100 (400 W), bench.py, ms/frame: 1 lane 25.4-25.5, 2 lanes 25.8 (one GPU has enough rays per wavefront; lanes are for small per-rank tile sets)
    CU(c->evFork.create(cudaEventCreateWithFlags, cudaEventDisableTiming));
    for (int l = 0; l < rtxpt_ctx::kMaxLanes; l++)
    {
        rtxpt_ctx::Lane& L = c->lanes[l];
        if (l > 0) CU(L.s.create(cudaStreamCreateWithFlags, cudaStreamNonBlocking));
        CU(L.s2.create(cudaStreamCreateWithFlags, cudaStreamNonBlocking));
        CU(L.evShadeDone.create(cudaEventCreateWithFlags, cudaEventDisableTiming)); CU(L.evShadowDone.create(cudaEventCreateWithFlags, cudaEventDisableTiming)); CU(L.evCommitted.create(cudaEventCreateWithFlags, cudaEventDisableTiming));
    }
    CU(c->hCounters.create(cudaHostAlloc<uint32_t>, kCounterWords * rtxpt_ctx::kMaxLanes * sizeof(uint32_t), cudaHostAllocDefault));
    memset(c->hCounters, 0, kCounterWords * rtxpt_ctx::kMaxLanes * sizeof(uint32_t));
    e = configureKernels(c->maxSmemOptin);
    if (e != cudaSuccess) return fail(RTXPT_ERR_CUDA, "kernel configuration failed: %s", cudaGetErrorString(e));
    {   // L2 persistence carve-out for the BVH nodes (off unless RTXPT_L2_PERSIST_MB is set; see DESIGN.md for the measurement)
        const char* e = getenv("RTXPT_L2_PERSIST_MB"); int maxPersist = 0, maxWindow = 0;
        cudaDeviceGetAttribute(&maxPersist, cudaDevAttrMaxPersistingL2CacheSize, c->device); cudaDeviceGetAttribute(&maxWindow, cudaDevAttrMaxAccessPolicyWindowSize, c->device);
        if (e && atoi(e) > 0 && maxPersist > 0)
        {
            c->l2PersistBytes = std::min(size_t(atoi(e)) << 20, size_t(maxPersist)); c->l2WindowMax = size_t(maxWindow);
            cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, c->l2PersistBytes);
        }
    }
    launchInitTables(c->stream);
    if ((e = cudaStreamSynchronize(c->stream)) != cudaSuccess) return fail(RTXPT_ERR_CUDA, "table initialisation failed: %s", cudaGetErrorString(e));
    *outCtx = c.release();
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_destroy(rtxpt_ctx* c)
{
    if (!c) return RTXPT_OK;
    cudaSetDevice(c->device);
    syncContext(c);
    delete c;
    return RTXPT_OK;
}

// ---- textures ----------------------------------------------------------------------------------------------------------------------
static bool isBlockCompressed(uint32_t format) { return format >= RTXPT_FORMAT_BC1_UNORM && format <= RTXPT_FORMAT_BC7_SRGB; }
static int createTexture2D(const RtxptTextureDesc& d, DeviceTexture& out)
{
    if (d.width == 0 || d.height == 0 || d.mipLevels == 0 || d.mipLevels > RTXPT_MAX_MIPS) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad texture description");
    if (d.format > RTXPT_FORMAT_BC7_SRGB) return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown texture format %u", d.format);
    const bool isFloat = d.format == RTXPT_FORMAT_RGBA32_FLOAT, isBc = isBlockCompressed(d.format);
    cudaChannelFormatDesc fmt = isFloat ? cudaCreateChannelDesc<float4>() : cudaCreateChannelDesc<uchar4>();
    size_t blockBytes = 0;
    if (isBc)
    {   // block-compressed array: the texture units decode BC1 / BC2 / BC3 / BC7 (and sRGB) on fetch, as the reference's TMUs do for its .dds assets
        if ((d.width & 3u) || (d.height & 3u)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "block-compressed textures need a width and height that are multiples of 4");
        switch (d.format)
        {
        case RTXPT_FORMAT_BC1_UNORM: fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed1>(); blockBytes = 8; break;
        case RTXPT_FORMAT_BC1_SRGB:  fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed1SRGB>(); blockBytes = 8; break;
        case RTXPT_FORMAT_BC2_UNORM: fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed2>(); blockBytes = 16; break;
        case RTXPT_FORMAT_BC2_SRGB:  fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed2SRGB>(); blockBytes = 16; break;
        case RTXPT_FORMAT_BC3_UNORM: fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed3>(); blockBytes = 16; break;
        case RTXPT_FORMAT_BC3_SRGB:  fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed3SRGB>(); blockBytes = 16; break;
        case RTXPT_FORMAT_BC7_UNORM: fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed7>(); blockBytes = 16; break;
        default:                     fmt = cudaCreateChannelDesc<cudaChannelFormatKindUnsignedBlockCompressed7SRGB>(); blockBytes = 16; break;
        }
    }
    CU(out.array.create(cudaMallocMipmappedArray, &fmt, make_cudaExtent(d.width, d.height, 0), d.mipLevels, 0u));
    const size_t texel = isFloat ? 16 : 4;
    for (uint32_t m = 0; m < d.mipLevels; m++)
    {
        cudaArray_t level; CU(cudaGetMipmappedArrayLevel(&level, out.array, m));
        const uint32_t w = std::max(1u, d.width >> m), h = std::max(1u, d.height >> m);
        if (!d.mips[m]) return fail(RTXPT_ERR_INVALID_ARGUMENT, "texture mip %u has no data", m);
        if (isBc) { const size_t rowBytes = size_t((w + 3) / 4) * blockBytes; CU(cudaMemcpy2DToArray(level, 0, 0, d.mips[m], rowBytes, rowBytes, (h + 3) / 4, cudaMemcpyHostToDevice)); }     // rows of blocks
        else CU(cudaMemcpy2DToArray(level, 0, 0, d.mips[m], w * texel, w * texel, h, cudaMemcpyHostToDevice));
    }
    cudaResourceDesc res{}; res.resType = cudaResourceTypeMipmappedArray; res.res.mipmap.mipmap = out.array;
    cudaTextureDesc td{};
    td.addressMode[0] = td.addressMode[1] = cudaAddressModeWrap;       // s_MaterialSampler: wrap, trilinear (CommonRenderPasses.cpp:85-86; anisotropy inert under SampleLevel)
    td.filterMode = cudaFilterModeLinear; td.mipmapFilterMode = cudaFilterModeLinear;
    td.readMode = isFloat ? cudaReadModeElementType : cudaReadModeNormalizedFloat;
    td.sRGB = (d.format == RTXPT_FORMAT_RGBA8_SRGB || d.format == RTXPT_FORMAT_BC1_SRGB || d.format == RTXPT_FORMAT_BC2_SRGB || d.format == RTXPT_FORMAT_BC3_SRGB || d.format == RTXPT_FORMAT_BC7_SRGB) ? 1 : 0;
    // (measured with scripts/probes/bc_probe.cu: the *SRGB block-compressed kinds are refused without td.sRGB, every block-compressed kind is refused with cudaReadModeElementType)
    td.normalizedCoords = 1; td.maxAnisotropy = 1; td.minMipmapLevelClamp = 0; td.maxMipmapLevelClamp = float(d.mipLevels - 1);
    CU(out.object.create(cudaCreateTextureObject, &res, &td, nullptr));
    td.filterMode = cudaFilterModePoint; td.mipmapFilterMode = cudaFilterModePoint;      // at a texel centre of an integer level: the texel itself, whatever the format
    CU(out.pointObject.create(cudaCreateTextureObject, &res, &td, nullptr));
    return RTXPT_OK;
}

// the layered, mipmapped float4 array of the environment cube and the texture object the kernels sample it through (filled by the caller)
static int allocEnvCube(uint32_t faceSize, uint32_t mipLevels, DeviceTexture& out)
{
    cudaChannelFormatDesc fmt = cudaCreateChannelDesc<float4>();
    CU(out.array.create(cudaMallocMipmappedArray, &fmt, make_cudaExtent(faceSize, faceSize, 6), mipLevels, cudaArrayLayered));
    cudaResourceDesc res{}; res.resType = cudaResourceTypeMipmappedArray; res.res.mipmap.mipmap = out.array;
    cudaTextureDesc td{};
    td.addressMode[0] = td.addressMode[1] = cudaAddressModeClamp; td.addressMode[2] = cudaAddressModeClamp;
    td.filterMode = cudaFilterModeLinear; td.mipmapFilterMode = cudaFilterModePoint; td.readMode = cudaReadModeElementType;
    td.normalizedCoords = 1; td.maxAnisotropy = 1; td.maxMipmapLevelClamp = float(mipLevels - 1);
    CU(out.object.create(cudaCreateTextureObject, &res, &td, nullptr));
    return RTXPT_OK;
}

static int createEnvCube(const RtxptEnvCubeDesc& d, DeviceTexture& out)
{
    if (d.mipLevels == 0 || d.mipLevels > RTXPT_MAX_MIPS) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad env cube description");
    int rc = allocEnvCube(d.faceSize, d.mipLevels, out); if (rc != RTXPT_OK) return rc;
    for (uint32_t m = 0; m < d.mipLevels; m++)
    {
        cudaArray_t level; CU(cudaGetMipmappedArrayLevel(&level, out.array, m));
        const uint32_t n = std::max(1u, d.faceSize >> m);
        for (int f = 0; f < 6; f++)
        {
            if (!d.faces[f][m]) return fail(RTXPT_ERR_INVALID_ARGUMENT, "env cube face %d mip %u has no data", f, m);
            cudaMemcpy3DParms cp{};
            cp.srcPtr = make_cudaPitchedPtr(const_cast<float*>(d.faces[f][m]), n * 16, n, n);
            cp.dstArray = level; cp.dstPos = make_cudaPos(0, 0, f); cp.extent = make_cudaExtent(n, n, 1); cp.kind = cudaMemcpyHostToDevice;
            CU(cudaMemcpy3D(&cp));
        }
    }
    return RTXPT_OK;
}

// ---- scene upload ----------------------------------------------------------------------------------------------------------------------
static inline void hostXformPoint(const float* m, const float* v, float* o)
{
    o[0] = m[0] * v[0] + m[1] * v[1] + m[2] * v[2] + m[3]; o[1] = m[4] * v[0] + m[5] * v[1] + m[6] * v[2] + m[7]; o[2] = m[8] * v[0] + m[9] * v[1] + m[10] * v[2] + m[11];
}

extern "C" RTXPT_API int rtxpt_b200_upload_scene(rtxpt_ctx* c, const RtxptSceneDesc* sc)
{
    if (!c || !sc) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    releaseScene(c);
    if (sc->materialCount > 0xFFFF || sc->textureCount > 0xFFFF || sc->bufferCount > 0xFFFF) return fail(RTXPT_ERR_UNSUPPORTED, "table sizes exceed the 16-bit indices of SubInstanceData");
    // validate + flatten triangles to world space (gid order: instance, geometry, primitive)
    std::vector<BuildTriangle> tris; std::vector<uint4> triInfo, triShade; std::vector<uint32_t> firstGid, maxVertex, prevPosBase; std::vector<float> triPrevPos;
    struct MaskJob { uint32_t tri, texture, cutoff; float uv[3][2]; }; std::vector<MaskJob> maskJobs;         // alpha-tested triangles that get an opacity mask (opacity_masks.h)
    const bool bakeMasks = !(c->cfg.flags & RTXPT_CFG_NO_OPACITY_MASKS);
    for (uint32_t ii = 0; ii < sc->instanceCount; ii++)
    {
        const RtxptInstanceData& inst = sc->instances[ii];
        for (uint32_t gi = 0; gi < inst.numGeometries; gi++)
        {
            if (inst.firstGeometryIndex + gi >= sc->geometryCount || inst.firstGeometryInstanceIndex + gi >= sc->subInstanceCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "instance %u references geometry out of range", ii);
            const RtxptGeometryData& g = sc->geometries[inst.firstGeometryIndex + gi];
            if (uint32_t(g.indexBufferIndex) >= sc->bufferCount || uint32_t(g.vertexBufferIndex) >= sc->bufferCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "geometry references buffer out of range");
            const uint32_t subIndex = inst.firstGeometryInstanceIndex + gi;
            if (firstGid.size() <= subIndex) firstGid.resize(size_t(subIndex) + 1, 0u);
            firstGid[subIndex] = uint32_t(tris.size());
            const bool hasPrev = g.prevPositionOffset != ~0u;          // Donut: only skinned geometries carry last frame's positions
            if (prevPosBase.size() <= subIndex) prevPosBase.resize(size_t(subIndex) + 1, 0xFFFFFFFFu);
            prevPosBase[subIndex] = hasPrev ? uint32_t(triPrevPos.size() / 9) : 0xFFFFFFFFu;
            if (maxVertex.size() <= subIndex) maxVertex.resize(size_t(subIndex) + 1, 0u);
            const RtxptSubInstanceData& sub = sc->subInstances[subIndex];
            uint32_t flags = subIndex;
            if (sub.FlagsAndAlphaInfo & RTXPT_SUBINST_FLAG_ALPHA_TESTED) flags |= kTriFlagAlphaTested;
            if (sub.FlagsAndAlphaInfo & RTXPT_SUBINST_FLAG_EXCLUDE_FROM_NEE) flags |= kTriFlagExcludeFromNEE;
            const uint8_t* ib = (const uint8_t*)sc->buffers[g.indexBufferIndex].data; const uint8_t* vb = (const uint8_t*)sc->buffers[g.vertexBufferIndex].data;
            const uint32_t triCount = g.numIndices / 3;
            if (uint64_t(g.indexOffset) + uint64_t(triCount) * 12 > sc->buffers[g.indexBufferIndex].sizeBytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "index range exceeds buffer");
            for (uint32_t t = 0; t < triCount; t++)
            {
                uint32_t idx[3]; memcpy(idx, ib + g.indexOffset + size_t(t) * 12, 12);
                maxVertex[subIndex] = std::max(maxVertex[subIndex], std::max(idx[0], std::max(idx[1], idx[2])));
                BuildTriangle bt; float* dst[3] = { bt.v0, bt.v1, bt.v2 };
                const uint64_t vbSize = sc->buffers[g.vertexBufferIndex].sizeBytes;
                uint4 rec[6]; memset(rec, 0, sizeof(rec));
                const bool hasUV = g.texCoord1Offset != ~0u, hasN = g.normalOffset != ~0u, hasT = g.tangentOffset != ~0u;
                for (int k = 0; k < 3; k++)
                {
                    if (uint64_t(g.positionOffset) + uint64_t(idx[k]) * 12 + 12 > vbSize) return fail(RTXPT_ERR_INVALID_ARGUMENT, "vertex index exceeds buffer");
                    if ((hasUV && uint64_t(g.texCoord1Offset) + uint64_t(idx[k]) * 8 + 8 > vbSize) || (hasN && uint64_t(g.normalOffset) + uint64_t(idx[k]) * 4 + 4 > vbSize) ||
                        (hasT && uint64_t(g.tangentOffset) + uint64_t(idx[k]) * 4 + 4 > vbSize)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "vertex attribute exceeds buffer");
                    float v[3]; memcpy(v, vb + g.positionOffset + size_t(idx[k]) * 12, 12);
                    hostXformPoint(inst.transform, v, dst[k]);
                    if (hasPrev)
                    {
                        if (uint64_t(g.prevPositionOffset) + uint64_t(idx[k]) * 12 + 12 > vbSize) return fail(RTXPT_ERR_INVALID_ARGUMENT, "previous-position stream exceeds buffer");
                        float pv[3]; memcpy(pv, vb + g.prevPositionOffset + size_t(idx[k]) * 12, 12); triPrevPos.insert(triPrevPos.end(), pv, pv + 3);
                    }
                    uint32_t w[3]; memcpy(w, v, 12); uint32_t nrm = 0, tan = 0, uv[2] = { 0, 0 };
                    if (hasN) memcpy(&nrm, vb + g.normalOffset + size_t(idx[k]) * 4, 4);
                    if (hasT) memcpy(&tan, vb + g.tangentOffset + size_t(idx[k]) * 4, 4);
                    if (hasUV) memcpy(uv, vb + g.texCoord1Offset + size_t(idx[k]) * 8, 8);
                    rec[k] = make_uint4(w[0], w[1], w[2], nrm);
                    if (k == 0) { rec[3].x = uv[0]; rec[3].y = uv[1]; rec[4].z = tan; }
                    if (k == 1) { rec[3].z = uv[0]; rec[3].w = uv[1]; rec[4].w = tan; }
                    if (k == 2) { rec[4].x = uv[0]; rec[4].y = uv[1]; rec[5].x = tan; }
                }
                if (t >= kTriShadePrimMask) return fail(RTXPT_ERR_UNSUPPORTED, "geometry with more than 2^29 triangles");
                rec[5].y = ii; rec[5].z = subIndex; rec[5].w = t | (hasUV ? kTriShadeHasUV : 0u) | (hasN ? kTriShadeHasNormal : 0u) | (hasT ? kTriShadeHasTangent : 0u);
                triShade.insert(triShade.end(), rec, rec + 6);
                bt.gid = uint32_t(tris.size()); bt.subInstanceAndFlags = flags; bt.primitiveIndex = om::kNoMask;       // third w word of the BVH triangle: opacity-mask slot
                if (bakeMasks && (flags & kTriFlagAlphaTested) && (sub.FlagsAndAlphaInfo & 0xFFFFu) < sc->textureCount)
                {
                    MaskJob j; j.tri = uint32_t(tris.size()); j.texture = sub.FlagsAndAlphaInfo & 0xFFFFu; j.cutoff = sub.FlagsAndAlphaInfo >> 24;
                    const uint32_t w[6] = { rec[3].x, rec[3].y, rec[3].z, rec[3].w, rec[4].x, rec[4].y }; memcpy(j.uv, w, 24);
                    maskJobs.push_back(j);
                }
                tris.push_back(bt);
                triInfo.push_back(make_uint4(ii, gi, t, subIndex));
            }
        }
    }
    if (tris.size() >= (size_t(1) << 27)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "scene has %zu triangles; the traversal kernels address at most 2^27 - 1", tris.size());
    // opacity masks: 64 two-bit states per alpha-tested triangle, baked from mip 0 of the alpha texture (the reference bakes OMMs for the same geometries, OmmBuildQueue.cpp:30-60)
    std::vector<uint4> masks(maskJobs.size()); uint64_t maskStates[3] = { 0, 0, 0 };
    std::vector<std::vector<uint8_t>> decodedAlpha(sc->textureCount);          // mip 0 of the block-compressed alpha textures, decoded once for the baker (the device keeps the blocks)
    for (const MaskJob& j : maskJobs)
    {
        const RtxptTextureDesc& td = sc->textures[j.texture];
        if (isBlockCompressed(td.format) && td.mips[0] && decodedAlpha[j.texture].empty()) rtxpt_host::decodeBlocksToRgba8(td.format, static_cast<const uint8_t*>(td.mips[0]), td.width, td.height, decodedAlpha[j.texture]);
    }
    {
        const auto t0 = std::chrono::steady_clock::now();
        #pragma omp parallel
        {
            uint32_t local[3] = { 0, 0, 0 };
            #pragma omp for schedule(dynamic, 256)
            for (int64_t i = 0; i < int64_t(maskJobs.size()); i++)
            {
                const MaskJob& j = maskJobs[size_t(i)]; const RtxptTextureDesc& td = sc->textures[j.texture];
                uint32_t m[4] = { 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu, 0xAAAAAAAAu };            // all unknown
                if (td.mips[0] && td.width && td.height)
                {
                    om::AlphaSource a; a.rgba8 = td.format == RTXPT_FORMAT_RGBA32_FLOAT ? nullptr : (isBlockCompressed(td.format) ? decodedAlpha[j.texture].data() : static_cast<const uint8_t*>(td.mips[0]));
                    a.rgba32f = td.format == RTXPT_FORMAT_RGBA32_FLOAT ? static_cast<const float*>(td.mips[0]) : nullptr; a.width = int(td.width); a.height = int(td.height);
                    om::bakeTriangle(a, j.cutoff, j.uv, m, local);
                }
                else local[om::kUnknown] += om::kMicroTriangles;
                masks[size_t(i)] = make_uint4(m[0], m[1], m[2], m[3]);
                tris[j.tri].primitiveIndex = uint32_t(i);
            }
            #pragma omp critical
            for (int k = 0; k < 3; k++) maskStates[k] += local[k];
        }
        c->opacityMaskTriangles = uint32_t(maskJobs.size()); for (int k = 0; k < 3; k++) c->opacityMaskStates[k] = maskStates[k];
        c->opacityMaskBakeSeconds = float(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count());
    }
    Bvh8 bvh;
    buildBvh8(tris, bvh);
    c->bvhBuildSeconds = float(bvh.buildSeconds);
    { const float dx = bvh.sceneHi[0] - bvh.sceneLo[0], dy = bvh.sceneHi[1] - bvh.sceneLo[1], dz = bvh.sceneHi[2] - bvh.sceneLo[2]; c->sceneDiagonal = tris.empty() ? 0.0f : sqrtf(dx * dx + dy * dy + dz * dz); }
    c->bvhNodeCount = uint32_t(bvh.nodes.size()); c->bvhTriCount = uint32_t(bvh.tris.size());
    for (int a = 0; a < 3; a++) { c->bvhRootBox[a] = bvh.sceneLo[a]; c->bvhRootBox[3 + a] = bvh.sceneHi[a]; }
    cudaStream_t s = c->stream;
    CU(c->dBvhNodes.upload(reinterpret_cast<const uint4*>(bvh.nodes.data()), bvh.nodes.size() * 5, s));
    CU(c->dBvhTris.upload(reinterpret_cast<const float4*>(bvh.tris.data()), bvh.tris.size() * 3, s));
    CU(c->dTriInfo.upload(triInfo.data(), triInfo.size(), s));
    CU(c->dTriShade.upload(triShade.data(), triShade.size(), s));
    prevPosBase.resize(std::max<size_t>(prevPosBase.size(), sc->subInstanceCount), 0xFFFFFFFFu);
    c->hPrevPosBase = prevPosBase; c->prevPosTriangles = triPrevPos.size() / 9;
    CU(c->dPrevPosBase.upload(prevPosBase.data(), prevPosBase.size(), s));
    CU(c->dTriPrevPos.upload(triPrevPos.data(), triPrevPos.size(), s));
    CU(c->dOpacityMasks.upload(masks.data(), masks.size(), s));
    CU(c->dInstances.upload(sc->instances, sc->instanceCount, s));
    c->hInstances.assign(sc->instances, sc->instances + sc->instanceCount); c->bvhLevelStart = bvh.levelStart; c->dNodeBox = {};
    c->hGeometries.assign(sc->geometries, sc->geometries + sc->geometryCount); c->firstGidOfSubInstance = firstGid; c->maxVertexOfSubInstance = maxVertex;
    CU(c->dGeometries.upload(sc->geometries, sc->geometryCount, s));
    CU(c->dMaterials.upload(sc->materials, sc->materialCount, s));
    c->materialCount = sc->materialCount;
    // bindless buffers
    std::vector<const uint8_t*> table(sc->bufferCount, nullptr);
    c->bufferAllocs.resize(sc->bufferCount);
    for (uint32_t i = 0; i < sc->bufferCount; i++) { CU(c->bufferAllocs[i].upload(static_cast<const uint8_t*>(sc->buffers[i].data), sc->buffers[i].sizeBytes, s)); table[i] = c->bufferAllocs[i].ptr; }
    CU(c->dBufferTable.upload(table.data(), table.size(), s));
    c->hBufferTable = table;
    // bindless textures
    std::vector<cudaTextureObject_t> texTable(sc->textureCount, 0);
    c->textures.resize(sc->textureCount);
    std::vector<cudaTextureObject_t> pointTable(sc->textureCount, 0); std::vector<uint4> texDims(sc->textureCount);
    for (uint32_t i = 0; i < sc->textureCount; i++)
    {
        int rc = createTexture2D(sc->textures[i], c->textures[i]); if (rc != RTXPT_OK) return rc;
        texTable[i] = c->textures[i].object; pointTable[i] = c->textures[i].pointObject;
        texDims[i] = make_uint4(sc->textures[i].width, sc->textures[i].height, sc->textures[i].mipLevels, 0u);
    }
    CU(c->dTextureTable.upload(texTable.data(), texTable.size(), s));
    CU(c->dPointTextureTable.upload(pointTable.data(), pointTable.size(), s));
    CU(c->dTextureDims.upload(texDims.data(), texDims.size(), s));
    c->envFaceSize = sc->envCube.faceSize; c->envMipLevels = sc->envCube.mipLevels;
    if (sc->envCube.faceSize) { int rc = createEnvCube(sc->envCube, c->envCube); if (rc != RTXPT_OK) return rc; }
    // sub-instances: shade-queue class (the SER sort key analogue; the reference sorts by material permutation, MaterialsBaker.cpp:1227-1285)
    c->hSubInstances.assign(sc->subInstances, sc->subInstances + sc->subInstanceCount);
    // AnalyticProxyLightIndex arrives as an index into sc->lights; in the light list the analytic lights follow the environment quad-tree nodes
    for (RtxptSubInstanceData& si : c->hSubInstances) si.AnalyticProxyLightIndex = (si.AnalyticProxyLightIndex < sc->lightCount) ? si.AnalyticProxyLightIndex + kEnvQuadLightCount : 0xFFFFFFFFu;
    // every enabled texture slot of every material must name an uploaded texture (the kernels index the bindless table without a bounds check, shade.cuh)
    for (uint32_t mi = 0; mi < sc->materialCount; mi++)
    {
        const RtxptMaterialData& m = sc->materials[mi];
        const struct { uint32_t flag, packed; const char* name; } slots[] = {
            { RTXPT_MATFLAG_UseBaseOrDiffuseTexture, m.BaseOrDiffuseTextureIndex, "base/diffuse" }, { RTXPT_MATFLAG_UseMetalRoughOrSpecularTexture, m.MetalRoughOrSpecularTextureIndex, "metal-rough/specular" },
            { RTXPT_MATFLAG_UseEmissiveTexture, m.EmissiveTextureIndex, "emissive" }, { RTXPT_MATFLAG_UseNormalTexture, m.NormalTextureIndex, "normal" },
            { RTXPT_MATFLAG_UseTransmissionTexture, m.TransmissionTextureIndex, "transmission" } };
        for (const auto& sl : slots)
            if ((m.Flags & sl.flag) && (sl.packed & 0xFFFFu) >= sc->textureCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "material %u: %s texture index %u out of range (%u textures)", mi, sl.name, sl.packed & 0xFFFFu, sc->textureCount);
    }
    std::vector<uint8_t> cls(sc->subInstanceCount, 0);
    for (uint32_t i = 0; i < sc->subInstanceCount; i++)
    {
        const uint32_t mi = c->hSubInstances[i].GlobalGeometryIndex_PTMaterialDataIndex & 0xFFFF;
        if (mi >= sc->materialCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "sub-instance %u references material out of range", i);
        const RtxptMaterialData& m = sc->materials[mi];
        if ((c->hSubInstances[i].FlagsAndAlphaInfo & RTXPT_SUBINST_FLAG_ALPHA_TESTED) && (c->hSubInstances[i].FlagsAndAlphaInfo & 0xFFFFu) >= sc->textureCount)
            return fail(RTXPT_ERR_INVALID_ARGUMENT, "alpha-tested sub-instance %u references texture %u of %u", i, c->hSubInstances[i].FlagsAndAlphaInfo & 0xFFFFu, sc->textureCount);
        const bool transmissive = m.TransmissionFactor > 0 || m.DiffuseTransmissionFactor > 0;
        const bool emissive = m.EmissiveColor[0] > 0 || m.EmissiveColor[1] > 0 || m.EmissiveColor[2] > 0;
        const bool textured = (m.Flags & (RTXPT_MATFLAG_UseBaseOrDiffuseTexture | RTXPT_MATFLAG_UseMetalRoughOrSpecularTexture | RTXPT_MATFLAG_UseNormalTexture | RTXPT_MATFLAG_UseEmissiveTexture)) != 0;
        cls[i] = transmissive ? 3 : (emissive ? 2 : (textured ? 1 : 0));
    }
    CU(c->dSubInstanceClass.upload(cls.data(), cls.size(), s));
    // lights (scene part); sub-instance table goes up after EmissiveLightMappingOffset is known
    LightBaker::prepareScene(*sc, c->hSubInstances, c->lightState);
    CU(c->dSubInstances.upload(c->hSubInstances.data(), c->hSubInstances.size(), s));
    CU(cudaStreamSynchronize(s));
    c->haveScene = true; c->lightsDirty = true; c->accumulatedSamples = 0;
    return RTXPT_OK;
}

// ---- constants -----------------------------------------------------------------------------------------------------------------------------
static int ensureTargets(rtxpt_ctx* c, uint32_t W, uint32_t H)
{
    if (W == 0 || H == 0 || W > 65535 || H > 65535) return fail(RTXPT_ERR_INVALID_ARGUMENT, "image size %ux%u unsupported (path id packs x,y in 16 bits each)", W, H);
    if (c->cfg.maxWidth && (W > c->cfg.maxWidth || H > c->cfg.maxHeight)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "image larger than the configured maximum");
    if (c->tableWidth == W && c->tableHeight == H) return RTXPT_OK;
    CU(syncContext(c));
    // pixels of this context's tiles, Morton order inside a tile: 32 consecutive path slots cover an 8x4 pixel block
    const uint32_t T = c->cfg.tileSize, tilesX = (W + T - 1) / T, tilesY = (H + T - 1) / T;
    std::vector<uint32_t> table;
    for (uint32_t t = c->cfg.tileRank; t < tilesX * tilesY; t += c->cfg.tileWorld)
    {
        const uint32_t tx = (t % tilesX) * T, ty = (t / tilesX) * T;
        for (uint32_t m = 0; m < T * T; m++)
        {
            uint32_t x = 0, y = 0;
            for (uint32_t b = 0; b < 16; b++) { x |= ((m >> (2 * b)) & 1u) << b; y |= ((m >> (2 * b + 1)) & 1u) << b; }
            if (tx + x < W && ty + y < H) table.push_back(((tx + x) << 16) | (ty + y));
        }
    }
    c->pixelCount = uint32_t(table.size());
    CU(c->pixelOfSlot.upload(table.data(), table.size(), c->stream));
    {   // pixel tables of every rank (deterministic from W,H,tileSize,world), padded to a common length: layout of the all-gather buffer
        std::vector<std::vector<uint32_t>> per(c->cfg.tileWorld);
        for (uint32_t t = 0; t < tilesX * tilesY; t++)
        {
            const uint32_t tx = (t % tilesX) * T, ty = (t / tilesX) * T;
            std::vector<uint32_t>& dst = per[t % c->cfg.tileWorld];
            for (uint32_t m = 0; m < T * T; m++)
            {
                uint32_t x = 0, y = 0;
                for (uint32_t b = 0; b < 16; b++) { x |= ((m >> (2 * b)) & 1u) << b; y |= ((m >> (2 * b + 1)) & 1u) << b; }
                if (tx + x < W && ty + y < H) dst.push_back(((tx + x) << 16) | (ty + y));
            }
        }
        size_t padded = 0; for (auto& v : per) padded = std::max(padded, v.size());
        c->paddedPixelsPerRank = uint32_t(padded);
        std::vector<uint32_t> all(padded * c->cfg.tileWorld, 0xFFFFFFFFu);
        for (uint32_t r = 0; r < c->cfg.tileWorld; r++) std::copy(per[r].begin(), per[r].end(), all.begin() + size_t(r) * padded);
        CU(c->allPixelTable.upload(all.data(), all.size(), c->stream));
    }
    const size_t P = size_t(W) * H;
    CU(c->outputColor.alloc(P)); CU(c->accumulated.alloc(P)); CU(c->depth.alloc(P)); CU(c->motionVectors.alloc(P)); CU(c->throughput.alloc(P));
    CU(c->motionVectors.fill(0, c->stream)); CU(c->throughput.fill(0, c->stream)); CU(c->outputColor.fill(0, c->stream)); CU(c->accumulated.fill(0, c->stream)); CU(c->depth.fill(0, c->stream));
    const size_t cap = size_t(c->pixelCount) * c->cfg.maxSubSamplesPerLaunch;
    if (cap >= 0x7FFFFFFFull) return fail(RTXPT_ERR_UNSUPPORTED, "too many path slots");
    c->capacity = uint32_t(std::max<size_t>(cap, 1));
    CU(c->s0.alloc(c->capacity)); CU(c->s1.alloc(c->capacity)); CU(c->s2.alloc(c->capacity)); CU(c->s3.alloc(c->capacity)); CU(c->s4.alloc(c->capacity));
    CU(c->t0.alloc(c->capacity)); CU(c->t1.alloc(c->capacity)); CU(c->t2.alloc(c->capacity)); CU(c->t3.alloc(c->capacity)); CU(c->t4.alloc(c->capacity)); CU(c->radiance.alloc(c->capacity));
    CU(c->hits.alloc(c->capacity)); CU(c->rayQueue[0].alloc(c->capacity)); CU(c->rayQueue[1].alloc(c->capacity));
    CU(c->shadeQueue.alloc(size_t(c->capacity) * kNumShadeClasses));
    CU(c->shadowOriginTMax.alloc(c->capacity)); CU(c->shadowDirPath.alloc(c->capacity)); CU(c->shadowRadiance.alloc(c->capacity));
    CU(c->counters.alloc(size_t(kCounterWords) * rtxpt_ctx::kMaxLanes));
    c->tableWidth = W; c->tableHeight = H; c->accumulatedSamples = 0;
    return RTXPT_OK;
}

static int uploadLights(rtxpt_ctx* c)
{
    LightBaker::finalize(c->consts, c->lightState);
    const LightBakeState& st = c->lightState;
    cudaStream_t s = c->stream;
    CU(cudaStreamSynchronize(s));
    CU(c->dLights.upload(reinterpret_cast<const LightInfo*>(st.lights.data()), st.lights.size(), s));
    CU(c->dProxyCounters.upload(st.proxyCounters.data(), st.proxyCounters.size(), s));
    if (!st.analyticLightsEx.empty()) CU(c->dLightsEx.upload(reinterpret_cast<const uint4*>(st.analyticLightsEx.data()), st.analyticLightsEx.size(), s));
    CU(c->dProxyIndices.upload(st.proxyIndices.data(), st.proxyIndices.size(), s));
    CU(c->dEnvLookup.upload(st.envLookupMap.data(), st.envLookupMap.size(), s));
    CU(cudaStreamSynchronize(s));
    c->lightsDirty = false; c->lightVersion++;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_set_constants(rtxpt_ctx* c, const RtxptPathTracerConstants* k)
{
    if (!c || !k) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    if (k->useApproximateMIS > 1) return fail(RTXPT_ERR_INVALID_ARGUMENT, "useApproximateMIS %u: 0 (full MIS) or 1 (approximate MIS)", k->useApproximateMIS);
    if (k->NEEFullSamples > 1 && k->NEEType == 2 && k->NEEATFeedback != 0)
        return fail(RTXPT_ERR_UNSUPPORTED, "NEEFullSamples > 1 together with NEE-AT temporal feedback is not supported: a visible sample's feedback draw decides the next sample's candidates, "
                                           "and the wavefront learns visibility only after the shadow kernel");
    if (k->bounceCount + 6 > (uint32_t)kMaxWavefrontIterations) return fail(RTXPT_ERR_UNSUPPORTED, "bounceCount above %d", kMaxWavefrontIterations - 6);
    int rc = ensureTargets(c, k->imageWidth, k->imageHeight);
    if (rc != RTXPT_OK) return rc;
    const bool envChanged = !c->haveConstants || memcmp(&c->consts.envMap, &k->envMap, sizeof(k->envMap)) != 0 || c->consts.distantVsLocalImportance != k->distantVsLocalImportance || c->consts.NEEType != k->NEEType;
    c->consts = *k; c->haveConstants = true;
    if (envChanged) c->lightsDirty = true;
    if (c->haveScene && c->lightsDirty) { rc = uploadLights(c); if (rc != RTXPT_OK) return rc; }
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_set_texture_filtering(rtxpt_ctx* c, const RtxptStochasticTextureFiltering* f)
{
    if (!c || !f) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (f->enable > 1) return fail(RTXPT_ERR_INVALID_ARGUMENT, "enable %u: 0 or 1", f->enable);
    if (f->filterType > RTXPT_STF_FILTER_TYPE_GAUSSIAN) return fail(RTXPT_ERR_INVALID_ARGUMENT, "filterType %u: STF_FILTER_TYPE_POINT (0) .. STF_FILTER_TYPE_GAUSSIAN (3)", f->filterType);
    if (!(std::isfinite(f->gaussianSigma) && f->gaussianSigma > 0.0f)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "gaussianSigma %g: finite and positive", double(f->gaussianSigma));
    if (f->magnificationMethod > 6) return fail(RTXPT_ERR_INVALID_ARGUMENT, "magnificationMethod %u: STF_MAGNIFICATION_METHOD_NONE (0) .. 4x4_FINE (6)", f->magnificationMethod);
    if (f->magnificationMethod != 0)
        return fail(RTXPT_ERR_UNSUPPORTED, "magnificationMethod %u: the wave magnification methods mix texels of whichever lanes share a wave, which the wavefront's sorted queues "
                                           "cannot reproduce; only STF_MAGNIFICATION_METHOD_NONE (0) is supported", f->magnificationMethod);
    c->stf = *f;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_set_debug_view(rtxpt_ctx* c, const RtxptDebugView* v)
{
    if (!c || !v) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    const uint32_t t = v->debugViewType;
    if (t >= RTXPT_DEBUG_VIEW_MAX_COUNT) return fail(RTXPT_ERR_INVALID_ARGUMENT, "debugViewType %u: DebugViewType has %u values", t, RTXPT_DEBUG_VIEW_MAX_COUNT);
    if (v->stablePlaneIndex >= RTXPT_STABLE_PLANE_COUNT && v->stablePlaneIndex != RTXPT_DEBUG_VIEW_STABLE_PLANE_SPLIT)
        return fail(RTXPT_ERR_INVALID_ARGUMENT, "stablePlaneIndex %u: 0..2 or RTXPT_DEBUG_VIEW_STABLE_PLANE_SPLIT", v->stablePlaneIndex);
    if (t >= RTXPT_DEBUG_VIEW_DENOISER_GUIDE_DEPTH && t <= RTXPT_DEBUG_VIEW_DENOISER_GUIDE_PRIMARY_LAYER)
        return fail(RTXPT_ERR_UNSUPPORTED, "debugViewType %u: the DenoiserGuide views read the DLSS-RR guide buffers, which this library does not produce", t);
    if (t >= RTXPT_DEBUG_VIEW_VBUFFER_MOTION_VECTORS)
        return fail(RTXPT_ERR_UNSUPPORTED, "debugViewType %u: the V-buffer, secondary-surface, ReSTIR and ReGIR views belong to RTXDI and the raster V-buffer, which this library does not have", t);
    c->debugView = *v;
    return RTXPT_OK;
}
// a call that draws a debug view starts from a cleared target.  RTXPT clears u_ShaderDebugVizTextureBuffer when the accumulation restarts (Sample.cpp:1427, under resetAccum);
// clearing on every call keeps a view from showing what an earlier call drew
static int clearDebugViz(rtxpt_ctx* c, cudaStream_t s)
{
    if (c->debugView.debugViewType == RTXPT_DEBUG_VIEW_DISABLED) return RTXPT_OK;
    const size_t P = size_t(c->tableWidth) * c->tableHeight;
    if (c->debugViz.count != P) { CU(syncContext(c)); CU(c->debugViz.alloc(P)); }
    CU(cudaMemsetAsync(c->debugViz.ptr, 0, P * sizeof(uint2), s));
    return RTXPT_OK;
}

// ---- launch --------------------------------------------------------------------------------------------------------------------------------
static void fillParams(rtxpt_ctx* c, LaunchParams& p)
{
    memset(&p, 0, sizeof(p));
    SceneView& v = p.scene;
    v.instances = c->dInstances.ptr; v.geometries = c->dGeometries.ptr; v.subInstances = c->dSubInstances.ptr; v.materials = c->dMaterials.ptr;
    v.subInstanceClass = c->dSubInstanceClass.ptr; v.materialCount = c->materialCount;
    v.buffers = c->dBufferTable.ptr; v.textures = c->dTextureTable.ptr; v.envCube = c->envCube.object; v.envFaceSize = c->envFaceSize; v.envMipLevels = c->envMipLevels;
    v.bvhNodes = c->dBvhNodes.ptr; v.bvhTris = c->dBvhTris.ptr; v.triInfo = c->dTriInfo.ptr; v.triShade = c->dTriShade.ptr; v.opacityMasks = c->dOpacityMasks.ptr; v.prevPosBase = c->dPrevPosBase.ptr; v.triPrevPos = c->dTriPrevPos.ptr; v.bvhNodeCount = c->bvhNodeCount; v.bvhTriCount = c->bvhTriCount;
    v.lightsEx = c->dLightsEx.ptr; v.analyticLightCount = uint32_t(c->lightState.analyticLightsEx.size());
    v.lights = c->dLights.ptr; v.proxyCounters = c->dProxyCounters.ptr; v.proxyIndices = c->dProxyIndices.ptr; v.envLookupMap = c->dEnvLookup.ptr;
    v.lightCount = uint32_t(c->lightState.lights.size()); v.samplingProxyCount = uint32_t(c->lightState.proxyIndices.size()); v.envEnabled = c->lightState.envEnabled ? 1u : 0u;
    WavefrontBuffers& w = p.wf;
    w.s0 = c->s0.ptr; w.s1 = c->s1.ptr; w.s2 = c->s2.ptr; w.s3 = c->s3.ptr; w.s4 = c->s4.ptr; w.hits = c->hits.ptr;
    w.rayQueue[0] = c->rayQueue[0].ptr; w.rayQueue[1] = c->rayQueue[1].ptr; w.shadeQueue = c->shadeQueue.ptr;
    w.shadowOriginTMax = c->shadowOriginTMax.ptr; w.shadowDirPath = c->shadowDirPath.ptr; w.shadowRadiance = c->shadowRadiance.ptr;
    w.counters = c->counters.ptr; w.pixelOfSlot = c->pixelOfSlot.ptr; w.capacity = c->capacity; w.pixelCount = c->pixelCount;
    p.stateIn = StateSet{ c->s0.ptr, c->s1.ptr, c->s2.ptr, c->s3.ptr, c->s4.ptr }; p.stateOut = StateSet{ c->t0.ptr, c->t1.ptr, c->t2.ptr, c->t3.ptr, c->t4.ptr }; p.radiance = c->radiance.ptr;
    if (c->stf.enable && c->dPointTextureTable.ptr)
    {   // stochastic texture filtering: the launchers pick the STF kernels when the table is set
        p.stf.pointTextures = c->dPointTextureTable.ptr; p.stf.textureDims = c->dTextureDims.ptr; p.stf.filterType = c->stf.filterType; p.stf.sigma = c->stf.gaussianSigma;
    }
    if (c->debugView.debugViewType != RTXPT_DEBUG_VIEW_DISABLED)
    {   // the launchers pick the debug-view kernels when the target is set; one active plane shows plane 0 (Sample.cpp:2161)
        p.dbg.viz = c->debugViz.ptr; p.dbg.view = c->debugView.debugViewType;
        p.dbg.planeIndex = (c->haveRealtime && c->realtime.activeStablePlaneCount == 1) ? 0 : int(c->debugView.stablePlaneIndex);
    }
    p.c = c->consts;
    p.flags = c->cfg.flags;
    p.refillThreshold = c->tune.refillThreshold; p.waitFlushLanes = c->tune.waitFlushLanes;
    p.shadowLongRayT = c->tune.shadowLpt ? 0.25f * c->sceneDiagonal : 3.0e38f;        // 3e38: every record goes to the back, i.e. one queue in reverse order
    p.outputColor = c->outputColor.ptr; p.accumulated = c->accumulated.ptr; p.depth = c->depth.ptr; p.motionVectors = c->motionVectors.ptr; p.throughput = c->throughput.ptr;
    memcpy(p.worldToClip, c->worldToClip, sizeof(p.worldToClip)); p.exportGuides = ((c->cfg.flags & RTXPT_CFG_EXPORT_GUIDES) && c->haveView) ? 1u : 0u;
    // traversal occupancy and the shared-memory BVH prefix are chosen together: B resident CTAs of 256 threads per SM (register budget
    // 65536 / (256 B): 128 / 85 / 64 registers for B = 2 / 3 / 4) share the 227 KB of shared memory
    const int blocks = c->tune.traceCtas;       // H100 (400 W), bench.py, ms/frame: 4 CTAs 25.4-25.5, 3 CTAs 26.7; shade CTAs (RTXPT_SHADE_CTAS): 3 25.6, 4 25.4-25.5, 5 27.3
    c->grid.traceBlocksPerSM = blocks;
    c->grid.shadeBlocksPerSM = c->tune.shadeCtas;
    const uint32_t budget = uint32_t(std::max(0, std::min(c->maxSmemOptin, (227 * 1024) / blocks - 2048) - 1024 - 8 * 2320));     // 8 x WarpScratch (traverse.cuh)
    // BVH prefix (breadth-first top levels) staged into shared memory by TMA: shared memory taken from the unified L1 costs the node and triangle
    // loads that miss the staged levels (H100 SXM, 700 W, bench.py: 200 staged nodes 23.72 ms/frame, none 23.16-23.18), so the default is 0 and RTXPT_SMEM_NODES opts in.
    // optional: keep the BVH nodes in the persisting part of L2 (RTXPT_L2_PERSIST_MB > 0) while path state streams through
    c->grid.l2WindowBase = nullptr; c->grid.l2WindowBytes = 0;
    if (c->l2PersistBytes && c->dBvhNodes.ptr) { c->grid.l2WindowBase = c->dBvhNodes.ptr; c->grid.l2WindowBytes = std::min(size_t(c->bvhNodeCount) * 80, c->l2WindowMax); c->grid.l2WindowHitRatio = std::min(1.0f, float(c->l2PersistBytes) / float(c->grid.l2WindowBytes)); }
    p.smemNodeCount = std::min(std::min(c->bvhNodeCount, budget / 80u), uint32_t(c->tune.smemNodes));
}

// RTXPT_CFG_TIME_KERNELS: bracket a launch with two events from the pool; kinds: 0 closest, 1 shadow, 2 shade, 3 other
struct KernelTimer
{
    rtxpt_ctx* c; cudaStream_t s; bool on;
    void begin(int kind)
    {
        if (!on) return;
        while (c->evPool.size() < c->evUsed + 2) { c->evPool.emplace_back(); c->evPool.back().create(cudaEventCreateWithFlags, cudaEventDefault); }
        c->evKind.resize(c->evPool.size() / 2 + 1); c->evKind[c->evUsed / 2] = kind;
        cudaEventRecord(c->evPool[c->evUsed], s);
    }
    void end() { if (!on) return; cudaEventRecord(c->evPool[c->evUsed + 1], s); c->evUsed += 2; }
};

static int checkReady(rtxpt_ctx* c)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    if (!c->haveConstants) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set");
    cudaSetDevice(c->device);
    if (c->lightsDirty) { int rc = uploadLights(c); if (rc != RTXPT_OK) return rc; }
    return RTXPT_OK;
}

// NEEFullSamples = N > 1: every vertex may emit N shadow records and owns an NEE block of 1 + N uint4, so a launch batches max(1, maxSubSamplesPerLaunch / N)
// sub-samples (include/rtxpt_b200.h) and the multi-sample arrays hold that many paths' records and blocks
static uint32_t neeFullSamples(const rtxpt_ctx* c) { return std::min(kNeeMaxFullSamples, c->consts.NEEFullSamples); }
static uint32_t multiSampleSubSamples(const rtxpt_ctx* c) { const uint32_t n = neeFullSamples(c); return n > 1 ? std::max(1u, c->cfg.maxSubSamplesPerLaunch / n) : c->cfg.maxSubSamplesPerLaunch; }
static int ensureNeeSamples(rtxpt_ctx* c)
{
    const uint32_t n = neeFullSamples(c);
    const size_t paths = size_t(multiSampleSubSamples(c)) * c->pixelCount, records = paths * n, blocks = paths * (1 + n);
    if (records >= 0x7FFFFFFFull || blocks >= 0xFFFFFFFFull) return fail(RTXPT_ERR_UNSUPPORTED, "NEEFullSamples %u: too many shadow records per launch", n);
    rtxpt_ctx::NeeSamples& a = c->neeSamples;
    if (a.originTMax.count >= records && a.blocks.count >= blocks) return RTXPT_OK;
    CU(syncContext(c));                 // earlier launches may still read the arrays being replaced
    cudaError_t e;
    if ((e = a.originTMax.alloc(records)) != cudaSuccess || (e = a.dirPath.alloc(records)) != cudaSuccess || (e = a.sample.alloc(records)) != cudaSuccess || (e = a.blocks.alloc(blocks)) != cudaSuccess)
    {   // nothing half-allocated stays behind, and the failed allocation is not reported again by a later launch: the context keeps rendering with fewer samples
        a = rtxpt_ctx::NeeSamples();
        cudaGetLastError();
        return fail(e == cudaErrorMemoryAllocation ? RTXPT_ERR_OUT_OF_MEMORY : RTXPT_ERR_CUDA, "NEEFullSamples %u: %zu shadow records and %zu NEE block words: %s", n, records, blocks, cudaGetErrorString(e));
    }
    return RTXPT_OK;
}
// point a launch's shadow records and NEE blocks at the multi-sample arrays, from path `first` on; the launch's p.wf.capacity paths own N records each (neeShadowCapacity)
static void useNeeSamples(rtxpt_ctx* c, LaunchParams& p, size_t first)
{
    const uint32_t n = neeFullSamples(c);
    WavefrontBuffers& w = p.wf;
    w.shadowOriginTMax = c->neeSamples.originTMax.ptr + first * n; w.shadowDirPath = c->neeSamples.dirPath.ptr + first * n; w.shadowRadiance = c->neeSamples.sample.ptr + first * n;
    p.neeBlocks = c->neeSamples.blocks.ptr + first * (1 + n);
}

static bool neeatActive(const rtxpt_ctx* c);
extern "C" RTXPT_API int rtxpt_b200_path_trace(rtxpt_ctx* c, uint32_t firstSubSampleIndex, uint32_t subSampleCount, int accumulate, void* cudaStream)
{
    int rc = checkReady(c); if (rc != RTXPT_OK) return rc;
    if (subSampleCount == 0) return RTXPT_OK;
    const bool na = neeatActive(c);
    if (na && (!c->na.allocated || !c->na.frameEnded)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEEATFeedback is set: call rtxpt_b200_neeat_update_begin and rtxpt_b200_neeat_update_end before tracing the frame");
    // tile partition (tileWorld > 1) with feedback: every rank adapts on the tiles it owns - independent global tables, reservoirs of foreign pixels stay empty (SURVEY §8e)
    if (na && !(c->cfg.flags & RTXPT_CFG_EXPORT_GUIDES)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEE-AT feedback in reference mode reprojects with the exported guides: create the context with RTXPT_CFG_EXPORT_GUIDES");
    cudaStream_t s = pickStream(c, cudaStream);
    rc = clearDebugViz(c, s); if (rc != RTXPT_OK) return rc;
    LaunchParams p; fillParams(c, p);
    if (na)
    {
        p.na = c->na.params; p.naShadowFeedback = c->na.shadowFeedback.ptr; p.naRrFix = c->na.rrFix.ptr;
        p.scene.proxyCounters = c->na.proxyCounters.ptr; p.scene.proxyIndices = c->na.proxyIndices.ptr;
    }
    const bool multi = neeFullSamples(c) > 1;          // (never together with feedback: rtxpt_b200_set_constants)
    if (multi) { rc = ensureNeeSamples(c); if (rc != RTXPT_OK) return rc; }
    // a pixel's feedback reservoir is updated by one path at a time, as in the reference's sequential sub-sample dispatches: no batching while feedback is active
    const uint32_t subSamplesPerLaunch = na ? 1u : multiSampleSubSamples(c);
    const TraceKind shadowKind = na ? TraceKind::ShadowNeeat : (multi ? TraceKind::ShadowMulti : TraceKind::Shadow);
    const bool countSteps = (c->cfg.flags & RTXPT_CFG_COUNT_TRAVERSAL_STEPS) != 0;
    const bool hasRefraction = c->consts.nestedDielectricsQuality > 0;
    const uint32_t iterations = std::min<uint32_t>(c->consts.bounceCount + 1 + (hasRefraction ? 4 : 0), kMaxWavefrontIterations);
    CU(cudaEventRecord(c->evStart, s));
    uint64_t launches = 0;
    KernelTimer kt{ c, s, (c->cfg.flags & RTXPT_CFG_TIME_KERNELS) != 0 };
    c->evUsed = 0;
    const bool overlap = c->overlapShadow && !kt.on;      // per-kernel timing wants the kernels back to back
    uint32_t lanesUsed = 1;
    for (uint32_t done = 0; done < subSampleCount; done += subSamplesPerLaunch)
    {
        const uint32_t n = std::min(subSamplesPerLaunch, subSampleCount - done);
        if (na) CU(cudaMemsetAsync(c->na.rrFix.ptr, 0, size_t(c->capacity) * 4, s));
        // pipeline lanes (see rtxpt_ctx::Lane): sub-samples [ first, first + count ) of this batch per lane; feedback (one path per pixel at a time) and per-kernel timing run one lane
        const uint32_t lanes = (na || kt.on) ? 1u : std::min<uint32_t>(uint32_t(c->tune.lanes), n);
        lanesUsed = lanes;
        CU(cudaMemsetAsync(c->counters.ptr, 0, size_t(kCounterWords) * lanes * sizeof(uint32_t), s));
        if (lanes > 1) CU(cudaEventRecord(c->evFork, s));
        for (uint32_t l = 0; l < lanes; l++)
        {
            const uint32_t firstSub = (l * n) / lanes, count = ((l + 1) * n) / lanes - firstSub;
            rtxpt_ctx::Lane& L = c->lanes[l];
            cudaStream_t ls = l == 0 ? s : L.s, ls2 = L.s2;
            if (l > 0) CU(cudaStreamWaitEvent(ls, c->evFork, 0));
            LaunchParams q = p;
            {   // the lane's slice of every per-path array: slots are lane-relative, pixel = slot mod pixelCount as before
                const size_t o = size_t(firstSub) * c->pixelCount; WavefrontBuffers& w = q.wf;
                w.s0 += o; w.s1 += o; w.s2 += o; w.s3 += o; w.s4 += o; w.hits += o; w.rayQueue[0] += o; w.rayQueue[1] += o; w.shadeQueue += o * kNumShadeClasses;
                w.shadowOriginTMax += o; w.shadowDirPath += o; w.shadowRadiance += o; w.counters += size_t(l) * kCounterWords; w.capacity = uint32_t(std::max<size_t>(size_t(count) * c->pixelCount, 1));
                if (na) { q.naShadowFeedback += o; q.naRrFix += o; }
                for (StateSet* st : { &q.stateIn, &q.stateOut }) { st->s0 += o; st->s1 += o; st->s2 += o; st->s3 += o; st->s4 += o; }
                q.radiance += o;
                if (multi) useNeeSamples(c, q, o);
            }
            q.firstSampleIndex = c->consts.sampleBaseIndex + firstSubSampleIndex + done + firstSub;
            q.subSampleCount = count;
            q.accumulatedSamples = c->accumulatedSamples + firstSub; q.doAccumulate = accumulate ? 1u : 0u;
            if (l + 1 != lanes) { q.exportGuides = 0; q.dbg.viz = nullptr; }     // the guides and the first-hit debug view hold the launch's last sub-sample, as after the reference's sequential dispatches
            if (done + n != subSampleCount) q.dbg.viz = nullptr;                  // the first-hit debug view holds the call's last sub-sample, whatever the launch split
            q.iteration = 0;
            KernelTimer ktl{ c, ls, kt.on };
            ktl.begin(3); launchGenerate(q, c->grid, ls); ktl.end(); launches++;
            // Shadow rays of vertex k and scatter rays of vertex k+1 touch disjoint state (shadow: shadow records + the path's radiance at its home index;
            // closest: ray words of the state set, hit records, shade queues), so k_trace_shadow(it) runs on a second stream next to k_trace_closest(it+1): the
            // long-ray tail of one persistent kernel is filled by the other's CTAs.  k_shade(it+1) joins both.
            for (uint32_t it = 0; it < iterations; it++)
            {
                q.iteration = it;
                if (it > 0) std::swap(q.stateIn, q.stateOut);     // the paths k_shade(it - 1) appended are iteration it's rays
                ktl.begin(0); launchTrace(TraceKind::Closest, q, c->grid, countSteps, ls); ktl.end();
                if (overlap && it > 0) CU(cudaStreamWaitEvent(ls, L.evShadowDone, 0));        // shadow(it-1) has updated the radiance words
                ktl.begin(2); if (na) launchShadeNeeat(q, c->grid, ls); else launchShade(q, c->grid, ls); ktl.end();
                if (overlap)
                {
                    CU(cudaEventRecord(L.evShadeDone, ls));
                    CU(cudaStreamWaitEvent(ls2, L.evShadeDone, 0));
                    launchTrace(shadowKind, q, c->grid, countSteps, ls2);
                    if (multi) launchNeeResolve(q, c->grid, false, ls2);          // the visible samples' radiance, before k_shade(it+1) reads it
                    CU(cudaEventRecord(L.evShadowDone, ls2));
                }
                else
                {
                    ktl.begin(1); launchTrace(shadowKind, q, c->grid, countSteps, ls); ktl.end();
                    if (multi) { ktl.begin(3); launchNeeResolve(q, c->grid, false, ls); ktl.end(); }
                }
                launches += multi ? 4 : 3;
            }
            if (overlap) CU(cudaStreamWaitEvent(ls, L.evShadowDone, 0));
            if (l > 0) CU(cudaStreamWaitEvent(ls, c->lanes[l - 1].evCommitted, 0));       // the running mean takes the sub-samples in order
            ktl.begin(3); launchCommitAccumulate(q, c->grid, ls); ktl.end(); launches++;
            if (lanes > 1) CU(cudaEventRecord(L.evCommitted, ls));
        }
        if (lanes > 1) CU(cudaStreamWaitEvent(s, c->lanes[lanes - 1].evCommitted, 0));     // every lane has committed (the commits are chained): the caller's stream joins
        if (accumulate) c->accumulatedSamples += n;
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(c->evStop, s));
    // statistics of the last batch (ray counts per iteration); read lazily by get_stats
    CU(cudaMemcpyAsync(c->hCounters, c->counters.ptr, size_t(kCounterWords) * lanesUsed * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    c->lastIterations = iterations; c->lastSubSamples = subSampleCount; c->lastLaunches = launches; c->lastLanes = lanesUsed; c->lastSubSamplesPerLaunch = subSamplesPerLaunch; c->statsPending = true;
    return RTXPT_OK;
}

static bool neeatActive(const rtxpt_ctx* c);
extern "C" RTXPT_API int rtxpt_b200_neeat_update_end(rtxpt_ctx* c, void* cudaStream);

// ---- realtime mode -----------------------------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API int rtxpt_b200_set_realtime(rtxpt_ctx* c, const RtxptRealtimeConstants* rt)
{
    if (!c || !rt) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveConstants) return fail(RTXPT_ERR_INVALID_ARGUMENT, "set the path tracer constants first (the image size sizes the plane buffers)");
    if (rt->activeStablePlaneCount < 1 || rt->activeStablePlaneCount > RTXPT_STABLE_PLANE_COUNT) return fail(RTXPT_ERR_INVALID_ARGUMENT, "activeStablePlaneCount must be 1..3");
    if (rt->subSampleCount < 1) return fail(RTXPT_ERR_INVALID_ARGUMENT, "subSampleCount must be at least 1");
    if (rt->maxStablePlaneVertexDepth > RTXPT_STABLE_PLANE_MAX_VERTEX_INDEX) return fail(RTXPT_ERR_INVALID_ARGUMENT, "maxStablePlaneVertexDepth above %u", RTXPT_STABLE_PLANE_MAX_VERTEX_INDEX);
    cudaSetDevice(c->device);
    const uint32_t W = c->tableWidth, H = c->tableHeight;
    if (c->realtimeWidth != W || c->realtimeHeight != H)
    {
        CU(syncContext(c));
        const size_t P = size_t(W) * H, planeStride = rtxpt_b200_generic_ts_plane_stride(W, H);
        CU(c->stablePlanes.alloc(planeStride * RTXPT_STABLE_PLANE_COUNT)); CU(c->stablePlanesHeader.alloc(P * 4)); CU(c->stableRadiance.alloc(P)); CU(c->specularHitT.alloc(P));
        CU(c->stablePlanes.fill(0, c->stream)); CU(c->stablePlanesHeader.fill(0xFF, c->stream)); CU(c->stableRadiance.fill(0, c->stream)); CU(c->specularHitT.fill(0, c->stream));
        c->realtimeWidth = W; c->realtimeHeight = H;
        c->realtimeFrameWidth = c->realtimeFrameHeight = 0;        // the new planes hold no frame yet
    }
    c->realtime = *rt; c->haveRealtime = true;
    return RTXPT_OK;
}

static void fillRealtimeParams(rtxpt_ctx* c, LaunchParams& p)
{
    const RtxptRealtimeConstants& r = c->realtime;
    p.rt.planes = c->stablePlanes.ptr; p.rt.header = c->stablePlanesHeader.ptr; p.rt.stableRadiance = c->stableRadiance.ptr; p.rt.specularHitT = c->specularHitT.ptr;
    p.rt.lineStride = rtxpt_b200_generic_ts_line_stride(c->tableWidth, c->tableHeight); p.rt.planeStride = rtxpt_b200_generic_ts_plane_stride(c->tableWidth, c->tableHeight);
    p.rt.activePlaneCount = r.activeStablePlaneCount; p.rt.maxVertexDepth = r.maxStablePlaneVertexDepth; p.rt.allowPSR = r.allowPrimarySurfaceReplacement;
    p.rt.attenuation = 1.0f / float(r.subSampleCount);
    memcpy(p.rt.worldToClipNoOffset, r.matWorldToClipNoOffset, 64); memcpy(p.rt.prevWorldToClipNoOffset, r.prevMatWorldToClipNoOffset, 64);
    p.rt.clipToWindowScale[0] = r.clipToWindowScale[0]; p.rt.clipToWindowScale[1] = r.clipToWindowScale[1];
    p.rt.dnViewZ = c->dnViewZ.ptr; p.rt.dnMotion = c->dnMotion.ptr; p.rt.dnNormalRoughness = c->dnNormalRoughness.ptr; p.rt.dnDiff = c->dnDiff.ptr; p.rt.dnSpec = c->dnSpec.ptr;
    p.rt.dnDisocclusionMix = c->dnDisocclusionMix.ptr; p.rt.dnHistoryClampRelax = c->dnHistoryClampRelax.ptr;
}
static int checkRealtimeReady(rtxpt_ctx* c)
{
    int rc = checkReady(c); if (rc != RTXPT_OK) return rc;
    if (!c->haveRealtime || c->realtimeWidth != c->tableWidth || c->realtimeHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_set_realtime has not been called for this image size");
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_path_trace_realtime(rtxpt_ctx* c, int mergeNoDenoiser, void* cudaStream)
{
    int rc = checkReady(c); if (rc != RTXPT_OK) return rc;
    if (!c->haveRealtime || c->realtimeWidth != c->tableWidth || c->realtimeHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_set_realtime has not been called for this image size");
    if (!c->haveView) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_set_view has not been called (the guide depth needs view.matWorldToClip)");
    cudaStream_t s = pickStream(c, cudaStream);
    const bool na = neeatActive(c);
    if (na && (!c->na.allocated || !c->na.frameBegun)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEEATFeedback is set: call rtxpt_b200_neeat_update_begin before tracing the frame");
    const bool multi = neeFullSamples(c) > 1;
    if (multi) { rc = ensureNeeSamples(c); if (rc != RTXPT_OK) return rc; }
    rc = clearDebugViz(c, s); if (rc != RTXPT_OK) return rc;
    LaunchParams p; fillParams(c, p);
    const RtxptRealtimeConstants& r = c->realtime;
    fillRealtimeParams(c, p);
    p.exportGuides = 0; p.subSampleCount = 1; p.doAccumulate = 0;
    const bool hasRefraction = c->consts.nestedDielectricsQuality > 0;
    // BUILD: the branches of a pixel's delta tree are explored one after the other, each at most maxVertexDepth + 1 segments long (+ rejected false hits)
    const uint32_t buildIterations = std::min<uint32_t>(r.activeStablePlaneCount * (std::min(r.maxStablePlaneVertexDepth, c->consts.bounceCount) + 1 + (hasRefraction ? 4 : 0)), kMaxWavefrontIterations);
    const uint32_t fillIterations = std::min<uint32_t>(c->consts.bounceCount + 1 + (hasRefraction ? 4 : 0), kMaxWavefrontIterations);
    CU(cudaEventRecord(c->evStart, s));
    uint64_t launches = 0;
    c->evUsed = 0;
    p.firstSampleIndex = c->consts.sampleBaseIndex;
    CU(cudaMemsetAsync(c->counters.ptr, 0, kCounterWords * sizeof(uint32_t), s));
    p.iteration = 0;
    launchRtBuildGenerate(p, c->grid, s); launches++;
    for (uint32_t it = 0; it < buildIterations; it++)
    {
        p.iteration = it;
        launchTrace(TraceKind::ClosestRealtime, p, c->grid, false, s); launchRtShade(p, c->grid, false, s); launches += 2;
    }
    if (na)
    {   // LightsBaker::UpdateEnd sits between the BUILD pass (this frame's depth and motion vectors) and the radiance passes (Sample.cpp:2495)
        rc = rtxpt_b200_neeat_update_end(c, cudaStream); if (rc != RTXPT_OK) return rc;
        p.na = c->na.params; p.naShadowFeedback = c->na.shadowFeedback.ptr; p.naRrFix = c->na.rrFix.ptr;
        p.scene.proxyCounters = c->na.proxyCounters.ptr; p.scene.proxyIndices = c->na.proxyIndices.ptr;
        launches += 4;
    }
    if (multi)
    {   // the FILL pass traces one path per pixel: the shade queues and the light samples' records are laid out for that many paths
        p.wf.capacity = std::max(c->pixelCount, 1u);
        useNeeSamples(c, p, 0);
    }
    for (uint32_t sub = 0; sub < r.subSampleCount; sub++)
    {
        p.firstSampleIndex = c->consts.sampleBaseIndex + sub;
        CU(cudaMemsetAsync(c->counters.ptr, 0, kCounterWords * sizeof(uint32_t), s));
        if (na) CU(cudaMemsetAsync(c->na.rrFix.ptr, 0, size_t(c->capacity) * 4, s));
        p.iteration = 0;
        launchRtFillGenerate(p, c->grid, s); launches++;
        for (uint32_t it = 0; it < fillIterations; it++)
        {
            p.iteration = it;
            launchTrace(TraceKind::ClosestRealtime, p, c->grid, false, s);
            if (na) { launchRtShadeNeeat(p, c->grid, s); launchTrace(TraceKind::ShadowRealtimeNeeat, p, c->grid, false, s); }
            else if (multi) { launchRtShade(p, c->grid, true, s); launchTrace(TraceKind::ShadowRealtimeMulti, p, c->grid, false, s); launchNeeResolve(p, c->grid, true, s); launches++; }
            else { launchRtShade(p, c->grid, true, s); launchTrace(TraceKind::ShadowRealtime, p, c->grid, false, s); }
            launches += 3;
        }
        launchRtFillCommit(p, c->grid, s); launches++;
    }
    if (p.dbg.viz && isStablePlaneView(p.dbg.view)) { launchRtDebugViz(p, c->grid, s); launches++; }      // StablePlanesDebugViz after the FILL pass (Sample.cpp:2551-2555)
    if (mergeNoDenoiser) { launchRtMerge(p, c->grid, s); launches++; }
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->evStop, s));
    CU(cudaMemcpyAsync(c->hCounters, c->counters.ptr, kCounterWords * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    c->lastIterations = fillIterations; c->lastSubSamples = 1; c->lastLaunches = launches; c->lastLanes = 1; c->lastSubSamplesPerLaunch = 1; c->statsPending = true;
    c->realtimeFrameWidth = c->tableWidth; c->realtimeFrameHeight = c->tableHeight;
    return RTXPT_OK;
}

// DenoisingGuidesBaker::DenoiseSpecHitT (Sample::PathTrace's "Denoising Guides Bake", Sample.cpp:2541-2543): ping guide -> scratch, pong scratch -> guide
extern "C" RTXPT_API int rtxpt_b200_denoise_spec_hit_t(rtxpt_ctx* c, void* cudaStream)
{
    int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
    cudaStream_t s = pickStream(c, cudaStream);
    const size_t P = size_t(c->tableWidth) * c->tableHeight;
    if (c->dnScratchFloat.count != P) { CU(syncContext(c)); CU(c->dnScratchFloat.alloc(P)); }
    launchDnSpecHitT(c->specularHitT.ptr, c->depth.ptr, c->dnScratchFloat.ptr, int(c->tableWidth), int(c->tableHeight), s);
    launchDnSpecHitT(c->dnScratchFloat.ptr, c->depth.ptr, c->specularHitT.ptr, int(c->tableWidth), int(c->tableHeight), s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}

// ---- RTXPT's side of the denoiser interface ------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API int rtxpt_b200_denoiser_prepare_inputs(rtxpt_ctx* c, uint32_t stablePlaneIndex, int initWithStableRadiance, const RtxptDenoiserConstants* k, void* cudaStream)
{
    int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
    if (!k || stablePlaneIndex >= RTXPT_STABLE_PLANE_COUNT) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad plane index or null constants");
    cudaStream_t s = pickStream(c, cudaStream);
    if (c->denoiserWidth != c->tableWidth || c->denoiserHeight != c->tableHeight)
    {
        CU(syncContext(c));
        const size_t P = size_t(c->tableWidth) * c->tableHeight;
        CU(c->dnViewZ.alloc(P)); CU(c->dnMotion.alloc(P)); CU(c->dnDiff.alloc(P)); CU(c->dnSpec.alloc(P)); CU(c->dnNormalRoughness.alloc(P)); CU(c->dnDisocclusionMix.alloc(P)); CU(c->dnHistoryClampRelax.alloc(P));
        CU(c->dnViewZ.fill(0, s)); CU(c->dnMotion.fill(0, s)); CU(c->dnDiff.fill(0, s)); CU(c->dnSpec.fill(0, s)); CU(c->dnNormalRoughness.fill(0, s)); CU(c->dnDisocclusionMix.fill(0, s)); CU(c->dnHistoryClampRelax.fill(0, s));
        c->denoiserWidth = c->tableWidth; c->denoiserHeight = c->tableHeight;
    }
    LaunchParams p; fillParams(c, p); fillRealtimeParams(c, p);
    p.rt.dn = *k; p.rt.dnPlane = stablePlaneIndex; p.rt.dnInitWithStableRadiance = initWithStableRadiance ? 1u : 0u;
    launchDnPrepareInputs(p, c->grid, s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}
// PostProcess DLSSRRDenoiserPrepareInputs (PostProcess.hlsl:175-440, Sample.cpp:2710-2757): the stable planes into the images DLSS Ray Reconstruction reads
extern "C" RTXPT_API int rtxpt_b200_dlss_rr_prepare_inputs(rtxpt_ctx* c, float brightnessClampK, void* cudaStream)
{
    int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
    if (c->realtimeFrameWidth != c->tableWidth || c->realtimeFrameHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "no realtime frame at this image size: run rtxpt_b200_path_trace_realtime first");
    if (!(std::isfinite(brightnessClampK) && brightnessClampK > 0.0f)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "DLSSRRBrightnessClampK must be finite and positive (RTXPT's default is 4096)");
    cudaStream_t s = pickStream(c, cudaStream);
    if (c->rrWidth != c->tableWidth || c->rrHeight != c->tableHeight)
    {
        CU(syncContext(c));
        const size_t P = size_t(c->tableWidth) * c->tableHeight;
        CU(c->rrDiffAlbedo.alloc(P)); CU(c->rrSpecAlbedo.alloc(P)); CU(c->rrNormalsRoughness.alloc(P)); CU(c->rrSpecMotionVectors.alloc(P));
        CU(c->rrDiffAlbedo.fill(0, s)); CU(c->rrSpecAlbedo.fill(0, s)); CU(c->rrNormalsRoughness.fill(0, s)); CU(c->rrSpecMotionVectors.fill(0, s));
        c->rrWidth = c->tableWidth; c->rrHeight = c->tableHeight;
    }
    LaunchParams p; fillParams(c, p); fillRealtimeParams(c, p);
    const DlssRrTargets rr{ c->rrDiffAlbedo.ptr, c->rrSpecAlbedo.ptr, c->rrNormalsRoughness.ptr, c->rrSpecMotionVectors.ptr, brightnessClampK };
    launchDnPrepareDlssRr(p, rr, c->grid, s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_denoiser_final_merge(rtxpt_ctx* c, uint32_t stablePlaneIndex, const void* dDiff, const void* dSpec, void* cudaStream)
{
    int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
    if (stablePlaneIndex >= RTXPT_STABLE_PLANE_COUNT) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad plane index");
    if (!dDiff && !dSpec)
    {   // NULL, NULL: the images rtxpt_b200_reblur_denoise wrote last
        if (c->reblurWidth != c->tableWidth || c->reblurHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "no denoised images: rtxpt_b200_reblur_denoise has not run");
        dDiff = c->rbOutDiff.ptr; dSpec = c->rbOutSpec.ptr;
    }
    if (!dDiff || !dSpec) return fail(RTXPT_ERR_INVALID_ARGUMENT, "one denoised image is null");
    if (c->denoiserWidth != c->tableWidth || c->denoiserHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_denoiser_prepare_inputs has not run (the sky mask lives in its view-space depth)");
    cudaStream_t s = pickStream(c, cudaStream);
    LaunchParams p; fillParams(c, p); fillRealtimeParams(c, p);
    p.rt.dnPlane = stablePlaneIndex; p.rt.dnDenoisedDiff = static_cast<const uint2*>(dDiff); p.rt.dnDenoisedSpec = static_cast<const uint2*>(dSpec);
    launchDnFinalMerge(p, c->grid, s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}

// ---- tone mapping (SURVEY §8f row 4) -------------------------------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API int rtxpt_b200_tone_map(rtxpt_ctx* c, const RtxptToneMappingParams* u, int sourceBuffer, void* cudaStream)
{
    if (!c || !u) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveConstants) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set (the image size comes from them)");
    if (u->toneMapOperator > 5) return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown tone-mapping operator %u", u->toneMapOperator);
    if (sourceBuffer != RTXPT_BUFFER_OUTPUT_COLOR_F16 && sourceBuffer != RTXPT_BUFFER_ACCUMULATED_F32) return fail(RTXPT_ERR_INVALID_ARGUMENT, "tone mapping reads the output colour or the accumulation buffer");
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    const size_t P = size_t(c->tableWidth) * c->tableHeight;
    if (c->ldrColor.count != P) { CU(syncContext(c)); CU(c->ldrColor.alloc(P)); CU(c->tmPartials.alloc(1024)); CU(c->tmAvgLuminance.alloc(1)); }
    const void* src = sourceBuffer == RTXPT_BUFFER_ACCUMULATED_F32 ? static_cast<const void*>(c->accumulated.ptr) : static_cast<const void*>(c->outputColor.ptr);
    if (!src) return fail(RTXPT_ERR_INVALID_ARGUMENT, "the source buffer does not exist yet");
    launchToneMap(tonemap::makeParams(*u), src, sourceBuffer == RTXPT_BUFFER_ACCUMULATED_F32, uint32_t(P), c->tmPartials.ptr, c->tmAvgLuminance.ptr, c->ldrColor.ptr, s);
    CU(cudaGetLastError());
    c->toneMapped = true;
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_tone_map_average_luminance(rtxpt_ctx* c, float* out)
{
    if (!c || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->toneMapped) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_tone_map has not run");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    CU(cudaMemcpy(out, c->tmAvgLuminance.ptr, 4, cudaMemcpyDeviceToHost));
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_tone_map_pre_exposed_gray(const RtxptToneMappingParams* u, float avgLuminance, float* outRgb)
{
    if (!u || !outRgb) return RTXPT_ERR_INVALID_ARGUMENT;
    tonemap::preExposedGray(*u, avgLuminance, outRgb);
    return RTXPT_OK;
}

// ---- rigid-instance animation: new instance matrices -> leaf triangles re-transformed, BVH refitted bottom-up (SURVEY §8f row 4; Sample.cpp:1170-1240) --------------------------
extern "C" RTXPT_API int rtxpt_b200_update_instance_transforms(rtxpt_ctx* c, const float* transforms3x4, uint32_t instanceCount, void* cudaStream)
{
    if (!c || !transforms3x4) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    if (instanceCount != c->hInstances.size()) return fail(RTXPT_ERR_INVALID_ARGUMENT, "expected %zu instance transforms, got %u", c->hInstances.size(), instanceCount);
    if (c->bvhTriCount == 0) return RTXPT_OK;
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    if (c->dNodeBox.count != size_t(c->bvhNodeCount) * 6) { CU(syncContext(c)); CU(c->dNodeBox.alloc(size_t(c->bvhNodeCount) * 6)); }
    for (uint32_t i = 0; i < instanceCount; i++)
    {   // Donut's InstanceData keeps last frame's matrix next to the current one (motion vectors of the BUILD pass read it)
        memcpy(c->hInstances[i].prevTransform, c->hInstances[i].transform, 48); memcpy(c->hInstances[i].transform, transforms3x4 + size_t(i) * 12, 48);
    }
    CU(cudaMemcpyAsync(c->dInstances.ptr, c->hInstances.data(), c->hInstances.size() * sizeof(RtxptInstanceData), cudaMemcpyHostToDevice, s));
    refit::Params p{};
    p.nodes = c->dBvhNodes.ptr; p.tris = c->dBvhTris.ptr; p.triShade = c->dTriShade.ptr; p.instances = c->dInstances.ptr; p.nodeBox = c->dNodeBox.ptr; p.nodeCount = c->bvhNodeCount; p.triCount = c->bvhTriCount;
    launchRefit(p, c->bvhLevelStart.data(), uint32_t(c->bvhLevelStart.size()) - 1, c->grid.smCount, s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}

// ---- device rebuild of the BVH over the current leaf triangles (bvh_build.cuh; what Sample::BuildTLAS / UpdateSkinnedBLASs ask of the driver every frame, Sample.cpp:1170-1240) ----
extern "C" RTXPT_API int rtxpt_b200_rebuild_bvh(rtxpt_ctx* c, void* cudaStream)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    const uint32_t n = c->bvhTriCount;
    if (n == 0) return RTXPT_OK;
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    rtxpt_ctx::BvhScratch& b = c->bvhScratch;
    const uint32_t tiles = (n + bvhb::kRadixTile - 1) / bvhb::kRadixTile;
    const size_t scanLen = std::max<size_t>(n, size_t(tiles) * 256), nodeCap = n;       // at most one wide node per BVH2 node with children (n - 1), or the root alone
    bool grown = false;
    auto grow = [&](auto& a, size_t count) -> cudaError_t {
        if (a.count >= count) return cudaSuccess;
        if (!grown) { grown = true; cudaError_t e = syncContext(c); if (e != cudaSuccess) return e; }
        return a.alloc(count);
    };
    CU(grow(b.tris, size_t(n) * 3)); CU(grow(b.outTris, size_t(n) * 3)); CU(grow(b.nodes, nodeCap * 5)); CU(grow(b.nodeBox, nodeCap * 6)); CU(grow(b.box2, size_t(n) * 12));
    for (int k = 0; k < 2; k++) { CU(grow(b.keys[k], n)); CU(grow(b.vals[k], n)); CU(grow(b.clusters[k], n)); }
    CU(grow(b.hist, size_t(tiles) * 256)); CU(grow(b.flags, n)); CU(grow(b.scanBlocks, (scanLen + kScanBlock - 1) / kScanBlock)); CU(grow(b.misc, 2));
    CU(grow(b.count2, size_t(n) * 2)); CU(grow(b.nn, n)); CU(grow(b.nodeRoot, nodeCap)); CU(grow(b.cenBounds, 6)); CU(grow(b.child2, n));
    if (!c->evBvhStart) { CU(c->evBvhStart.create(cudaEventCreateWithFlags, cudaEventDefault)); CU(c->evBvhStop.create(cudaEventCreateWithFlags, cudaEventDefault)); }
    bvhb::Params p{};
    p.srcTris = c->dBvhTris.ptr; p.tris = b.tris.ptr; p.triCount = n; p.cenBounds = b.cenBounds.ptr; p.varying = b.misc.ptr + 1;
    for (int k = 0; k < 2; k++) { p.keys[k] = b.keys[k].ptr; p.vals[k] = b.vals[k].ptr; p.clusters[k] = b.clusters[k].ptr; }
    p.hist = b.hist.ptr; p.box2 = b.box2.ptr; p.child2 = b.child2.ptr; p.count2 = b.count2.ptr; p.nn = b.nn.ptr; p.flags = b.flags.ptr;
    p.nodeRoot = b.nodeRoot.ptr; p.levelCounts = b.flags.ptr;          // the PLOC flags are dead once the clustering is done
    p.nodes = b.nodes.ptr; p.outTris = b.outTris.ptr; p.nodeBox = b.nodeBox.ptr;
    CU(cudaEventRecord(c->evBvhStart, s));
    BvhBuildResult r;
    CU(launchBvhBuild(p, BvhBuildScans{ b.scanBlocks.ptr, b.misc.ptr }, c->grid.smCount, s, r));
    if (r.status == BvhBuildResult::kTooDeep) return fail(RTXPT_ERR_UNSUPPORTED, "rebuilt BVH would be deeper than %u levels (traversal stack); the previous tree is kept", bvhb::kMaxDepth);
    if (r.status != BvhBuildResult::kOk) return fail(RTXPT_ERR_INTERNAL, "BVH rebuild did not converge; the previous tree is kept");
    CU(cudaEventRecord(c->evBvhStop, s)); CU(cudaEventSynchronize(c->evBvhStop));
    float ms = 0; CU(cudaEventElapsedTime(&ms, c->evBvhStart, c->evBvhStop));
    std::swap(c->dBvhNodes, b.nodes); std::swap(c->dBvhTris, b.outTris);
    c->bvhNodeCount = r.nodeCount; c->bvhLevelStart = r.levelStart; c->dNodeBox = {};
    for (int a = 0; a < 6; a++) c->bvhRootBox[a] = r.rootBox[a];
    { const float dx = r.rootBox[3] - r.rootBox[0], dy = r.rootBox[4] - r.rootBox[1], dz = r.rootBox[5] - r.rootBox[2]; c->sceneDiagonal = sqrtf(dx * dx + dy * dy + dz * dz); }
    c->bvhBuildSeconds = ms * 1e-3f;
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_get_bvh_stats(rtxpt_ctx* c, RtxptBvhStats* out)
{
    if (!c || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    cudaSetDevice(c->device);
    memset(out, 0, sizeof(*out));
    out->nodeCount = c->bvhNodeCount; out->triangleReferenceCount = c->bvhTriCount; out->maxDepth = uint32_t(c->bvhLevelStart.size()) - 1; out->buildSeconds = c->bvhBuildSeconds;
    if (c->bvhTriCount == 0) return RTXPT_OK;
    CU(syncContext(c));
    std::vector<Bvh8Node> nodes(c->bvhNodeCount);
    CU(cudaMemcpy(nodes.data(), c->dBvhNodes.ptr, nodes.size() * sizeof(Bvh8Node), cudaMemcpyDeviceToHost));
    float root[6]; memcpy(root, c->bvhRootBox, 24);
    if (c->dNodeBox.count >= 6) CU(cudaMemcpy(root, c->dNodeBox.ptr, 24, cudaMemcpyDeviceToHost));     // refitted since the last build: the root's exact box now
    double visits = 0, tests = 0;
    bvh8SahStats(nodes.data(), nodes.size(), root, root + 3, &visits, &tests, &out->leafCount);
    out->expectedNodeVisits = float(visits); out->expectedTriangleTests = float(tests);
    return RTXPT_OK;
}

// ---- skinned meshes (SURVEY §8f row 4): Donut's skinning pass + the rewrite of the path tracer's per-triangle shade records; the caller refits afterwards -----------------------
extern "C" RTXPT_API int rtxpt_b200_skin_register(rtxpt_ctx* c, const RtxptSkinDesc* d, uint32_t* outSkinId)
{
    if (!c || !d || !outSkinId) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    if (d->instanceIndex >= c->hInstances.size() || d->geometryIndexInInstance >= c->hInstances[d->instanceIndex].numGeometries) return fail(RTXPT_ERR_INVALID_ARGUMENT, "instance / geometry out of range");
    if (!d->positions || !d->jointIndices || !d->jointWeights || d->numVertices == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bind pose needs positions, joint indices and weights");
    const RtxptInstanceData& inst = c->hInstances[d->instanceIndex];
    const RtxptGeometryData& g = c->hGeometries[inst.firstGeometryIndex + d->geometryIndexInInstance];
    if (d->numVertices != g.numVertices && g.numVertices != 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "geometry has %u vertices, bind pose %u", g.numVertices, d->numVertices);
    // the bind pose must cover every vertex the geometry's triangles name and every joint a non-zero weight names (the kernels index without bounds checks, skinning.cuh)
    uint32_t maxJoint = 0, maxIndex = 0;
    for (size_t v = 0; v < size_t(d->numVertices) * 4; v++) if (d->jointWeights[v] > 0.0f) maxJoint = std::max<uint32_t>(maxJoint, d->jointIndices[v]);
    maxIndex = c->maxVertexOfSubInstance[inst.firstGeometryInstanceIndex + d->geometryIndexInInstance];
    if (g.numIndices && maxIndex >= d->numVertices) return fail(RTXPT_ERR_INVALID_ARGUMENT, "geometry indexes vertex %u, bind pose has %u vertices", maxIndex, d->numVertices);
    cudaSetDevice(c->device);
    cudaStream_t s = c->stream;
    auto sk = std::make_unique<rtxpt_ctx::Skin>();
    sk->maxJoint = maxJoint;
    sk->numVertices = d->numVertices; sk->numTriangles = g.numIndices / 3; sk->firstGid = c->firstGidOfSubInstance[inst.firstGeometryInstanceIndex + d->geometryIndexInInstance];
    sk->flags = (d->normals ? 2u : 0u) | (d->tangents ? 4u : 0u);
    sk->dIndices = reinterpret_cast<const uint32_t*>(c->hBufferTable[g.indexBufferIndex] + g.indexOffset);
    CU(sk->positions.upload(d->positions, size_t(d->numVertices) * 3, s)); CU(sk->jointIndices.upload(d->jointIndices, size_t(d->numVertices) * 4, s)); CU(sk->weights.upload(d->jointWeights, size_t(d->numVertices) * 4, s));
    if (d->normals) CU(sk->normals.upload(d->normals, d->numVertices, s));
    if (d->tangents) CU(sk->tangents.upload(d->tangents, d->numVertices, s));
    CU(sk->outPositions.alloc(size_t(d->numVertices) * 3)); CU(sk->outNormals.alloc(d->numVertices)); CU(sk->outTangents.alloc(d->numVertices));
    CU(cudaStreamSynchronize(s));
    {   // last frame's positions for the BUILD pass's motion vectors: a geometry that came without a previous-position stream gets a range now, holding its current corners
        const uint32_t subIndex = inst.firstGeometryInstanceIndex + d->geometryIndexInInstance;
        if (c->hPrevPosBase[subIndex] == 0xFFFFFFFFu && sk->numTriangles)
        {
            CU(syncContext(c));
            DeviceArray<float> grown;
            CU(grown.alloc((c->prevPosTriangles + sk->numTriangles) * 9));
            if (c->prevPosTriangles) CU(cudaMemcpy(grown.ptr, c->dTriPrevPos.ptr, c->prevPosTriangles * 36, cudaMemcpyDeviceToDevice));
            c->dTriPrevPos = std::move(grown);
            c->hPrevPosBase[subIndex] = uint32_t(c->prevPosTriangles); c->prevPosTriangles += sk->numTriangles;
            CU(cudaMemcpy(c->dPrevPosBase.ptr + subIndex, &c->hPrevPosBase[subIndex], 4, cudaMemcpyHostToDevice));
            skin::Params ip{}; ip.numTriangles = sk->numTriangles; ip.firstGid = sk->firstGid; ip.triShade = c->dTriShade.ptr; ip.triPrevPos = c->dTriPrevPos.ptr + size_t(c->hPrevPosBase[subIndex]) * 9;
            launchSkinInitPrev(ip, s); CU(cudaStreamSynchronize(s));
        }
        sk->prevPosFirst = c->hPrevPosBase[subIndex];
    }
    c->skins.push_back(std::move(sk)); *outSkinId = uint32_t(c->skins.size() - 1);
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_skin_update(rtxpt_ctx* c, uint32_t skinId, const float* jointMatrices4x4, uint32_t numJoints, void* cudaStream)
{
    if (!c || !jointMatrices4x4) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (skinId >= c->skins.size()) return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown skin %u", skinId);
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    rtxpt_ctx::Skin& sk = *c->skins[skinId];
    if (numJoints <= sk.maxJoint) return fail(RTXPT_ERR_INVALID_ARGUMENT, "skin %u uses joint %u, %u joint matrices given", skinId, sk.maxJoint, numJoints);
    if (sk.jointMatrices.count != size_t(numJoints) * 16) { CU(cudaStreamSynchronize(s)); CU(sk.jointMatrices.alloc(size_t(numJoints) * 16)); }
    CU(cudaMemcpyAsync(sk.jointMatrices.ptr, jointMatrices4x4, size_t(numJoints) * 64, cudaMemcpyHostToDevice, s));
    sk.numJoints = numJoints;
    skin::Params p{};
    p.numVertices = sk.numVertices; p.numTriangles = sk.numTriangles; p.firstGid = sk.firstGid; p.flags = sk.flags;
    p.positions = sk.positions.ptr; p.normals = sk.normals.ptr; p.tangents = sk.tangents.ptr; p.jointIndices = sk.jointIndices.ptr; p.jointWeights = sk.weights.ptr; p.jointMatrices = sk.jointMatrices.ptr;
    p.outPositions = sk.outPositions.ptr; p.outNormals = sk.outNormals.ptr; p.outTangents = sk.outTangents.ptr; p.indices = sk.dIndices; p.triShade = c->dTriShade.ptr;
    p.triPrevPos = c->dTriPrevPos.ptr + size_t(sk.prevPosFirst) * 9;
    launchSkin(p, s);
    CU(cudaGetLastError());
    return RTXPT_OK;
}
// tests / debugging: the scene state the refit and skinning kernels write (include/rtxpt_b200.h lists the `what` codes); dst == NULL returns the size only
extern "C" RTXPT_API int rtxpt_b200_debug_scene_readback(rtxpt_ctx* c, int what, void* dst, size_t dstBytes, size_t* outBytes)
{
    if (!c || !outBytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    const void* src = nullptr; size_t bytes = 0; bool host = false;
    switch (what)
    {
    case 0: src = c->dBvhNodes.ptr; bytes = size_t(c->bvhNodeCount) * 80; break;
    case 1: src = c->dBvhTris.ptr; bytes = size_t(c->bvhTriCount) * 48; break;
    case 2: src = c->dTriShade.ptr; bytes = c->dTriShade.count * sizeof(uint4); break;
    case 3: src = c->dTriPrevPos.ptr; bytes = c->prevPosTriangles * 36; break;
    case 4: src = c->dInstances.ptr; bytes = c->hInstances.size() * sizeof(RtxptInstanceData); break;
    case 5: src = c->bvhLevelStart.data(); bytes = c->bvhLevelStart.size() * 4; host = true; break;
    case 6: src = c->dNodeBox.ptr; bytes = c->dNodeBox.count * 4; break;
    case 7: if (c->envCube.array) for (uint32_t m = 0; m < c->envMipLevels; m++) bytes += size_t(6) * (c->envFaceSize >> m) * (c->envFaceSize >> m) * 16; break;
    case 8: for (const std::vector<float>& mip : c->lightState.envRadianceMips) bytes += mip.size() * 4; break;
    case 9: src = c->dEnvLookup.ptr; bytes = c->dEnvLookup.count * 4; break;
    default: return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown scene buffer %d", what);
    }
    *outBytes = bytes;
    if (!dst || bytes == 0) return RTXPT_OK;
    if (dstBytes < bytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "destination too small (%zu < %zu)", dstBytes, bytes);
    if (what == 7)
    {   // the cube array, MIP by MIP, six faces back to back (the layout rtxpt_b200_bake_env_map returns)
        size_t off = 0;
        for (uint32_t m = 0; m < c->envMipLevels; m++)
        {
            const uint32_t n = c->envFaceSize >> m;
            cudaArray_t level; CU(cudaGetMipmappedArrayLevel(&level, c->envCube.array, m));
            cudaMemcpy3DParms cp{};
            cp.srcArray = level; cp.dstPtr = make_cudaPitchedPtr(static_cast<uint8_t*>(dst) + off, size_t(n) * 16, n, n); cp.extent = make_cudaExtent(n, n, 6); cp.kind = cudaMemcpyDeviceToHost;
            CU(cudaMemcpy3D(&cp));
            off += size_t(6) * n * n * 16;
        }
    }
    else if (what == 8) { size_t off = 0; for (const std::vector<float>& mip : c->lightState.envRadianceMips) { memcpy(static_cast<uint8_t*>(dst) + off, mip.data(), mip.size() * 4); off += mip.size() * 4; } }
    else if (host) memcpy(dst, src, bytes); else CU(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    return RTXPT_OK;
}

// ---- environment-map baking (SURVEY §8f row 3) ---------------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API uint32_t rtxpt_b200_env_bake_mip_count(uint32_t cubeDim) { uint32_t l = 0; while ((cubeDim >> l) > 0) l++; return l; }
extern "C" RTXPT_API size_t rtxpt_b200_env_bake_floats(uint32_t cubeDim) { size_t n = 0; for (uint32_t m = 0; (cubeDim >> m) > 0; m++) n += size_t(6) * (cubeDim >> m) * (cubeDim >> m) * 4; return n; }
// what rtxpt_b200_bake_env_map and rtxpt_b200_update_env_map accept; `sourceMayBeKept`: a cube or equirectangular source may come without pixels (the context's kept source)
static int checkEnvBakeDesc(const RtxptEnvBakeDesc* d, bool sourceMayBeKept)
{
    if (d->cubeDim < 2 || d->cubeDim > 4096 || (d->cubeDim & (d->cubeDim - 1))) return fail(RTXPT_ERR_INVALID_ARGUMENT, "cubeDim must be a power of two in 2..4096");
    if (d->directionalLightCount > 16) return fail(RTXPT_ERR_INVALID_ARGUMENT, "at most 16 directional lights (EMB_MAXDIRLIGHTS)");
    if (d->sourceType > 2 || (d->sourceType != 0 && ((!d->source && !sourceMayBeKept) || d->sourceWidth == 0 || (d->sourceType == 1 && d->sourceHeight == 0)))) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad source description");
    return RTXPT_OK;
}
static size_t envSourceFloats(const RtxptEnvBakeDesc* d) { return d->sourceType == 1 ? size_t(d->sourceWidth) * d->sourceHeight * 4 : (d->sourceType == 2 ? size_t(6) * d->sourceWidth * d->sourceWidth * 4 : 0); }
// the bake of `d` from `source` (device, NULL without one) into `mips`: all MIPs back to back, rtxpt_b200_env_bake_floats(cubeDim) floats
static envbake::Params envBakeParams(const RtxptEnvBakeDesc* d, const float* source, float* mips)
{
    envbake::Params p{};
    p.cubeDim = d->cubeDim; p.sourceType = d->sourceType; p.sourceWidth = d->sourceWidth; p.sourceHeight = d->sourceHeight; p.source = source;
    memcpy(p.scaleColor, d->scaleColor, 12); p.lightCount = d->directionalLightCount;
    for (uint32_t i = 0; i < d->directionalLightCount; i++) { memcpy(p.lights[i].colorIntensity, d->lights[i].colorIntensity, 16); memcpy(p.lights[i].direction, d->lights[i].direction, 12); p.lights[i].angularSize = d->lights[i].angularSize; }
    size_t off = 0; for (uint32_t m = 0; m < rtxpt_b200_env_bake_mip_count(d->cubeDim); m++) { p.mips[m] = mips + off; off += size_t(6) * (d->cubeDim >> m) * (d->cubeDim >> m) * 4; }
    return p;
}
extern "C" RTXPT_API int rtxpt_b200_bake_env_map(rtxpt_ctx* c, const RtxptEnvBakeDesc* d, float* out, size_t outFloats)
{
    if (!c || !d || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    int rc = checkEnvBakeDesc(d, false); if (rc != RTXPT_OK) return rc;
    const size_t total = rtxpt_b200_env_bake_floats(d->cubeDim);
    if (outFloats < total) return fail(RTXPT_ERR_INVALID_ARGUMENT, "output too small (%zu < %zu floats)", outFloats, total);
    cudaSetDevice(c->device);
    cudaStream_t s = c->stream;
    const uint32_t levels = rtxpt_b200_env_bake_mip_count(d->cubeDim);
    DeviceArray<float> src, dst;
    const size_t srcFloats = envSourceFloats(d);
    if (srcFloats) CU(src.upload(d->source, srcFloats, s));
    CU(dst.alloc(total));
    launchEnvBake(envBakeParams(d, src.ptr, dst.ptr), levels, s);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, dst.ptr, total * 4, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return RTXPT_OK;
}

// EnvMapBaker::Update with contentsChanged, then EnvMapImportanceSamplingBaker and the environment passes of LightsBaker (Sample.cpp, UpdateLighting): the bake goes straight into
// the cube the kernels sample, the importance map is built on the GPU from it, and the host light bake builds the quad-tree lights from that map
extern "C" RTXPT_API int rtxpt_b200_update_env_map(rtxpt_ctx* c, const RtxptEnvBakeDesc* d, void* cudaStream)
{
    if (!c || !d) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    int rc = checkEnvBakeDesc(d, true); if (rc != RTXPT_OK) return rc;
    const bool keptSource = d->sourceType != 0 && !d->source;
    if (keptSource && (!c->envSource.ptr || c->envSourceType != d->sourceType || c->envSourceWidth != d->sourceWidth || (d->sourceType == 1 && c->envSourceHeight != d->sourceHeight)))
        return fail(RTXPT_ERR_INVALID_ARGUMENT, "no kept source of type %u and size %ux%u to re-bake from", d->sourceType, d->sourceWidth, d->sourceType == 1 ? d->sourceHeight : d->sourceWidth);
    cudaSetDevice(c->device);
    CU(syncContext(c));
    cudaStream_t s = pickStream(c, cudaStream);
    const uint32_t dim = d->cubeDim, levels = rtxpt_b200_env_bake_mip_count(dim);
    const size_t bakeFloats = rtxpt_b200_env_bake_floats(dim);
    size_t importanceFloats = 0; for (uint32_t m = 0; m < envbake::kImportanceMips; m++) importanceFloats += size_t(envbake::kImportanceDim >> m) * (envbake::kImportanceDim >> m) * 4;
    if (c->envBakeScratch.count < bakeFloats) CU(c->envBakeScratch.alloc(bakeFloats));
    if (c->envImportanceScratch.count < importanceFloats) CU(c->envImportanceScratch.alloc(importanceFloats));
    if (!c->evEnv[0]) for (Event& e : c->evEnv) CU(e.create(cudaEventCreateWithFlags, cudaEventDefault));
    DeviceArray<float> fresh;         // a new source replaces the kept one once the update has succeeded
    if (d->sourceType != 0 && !keptSource) CU(fresh.upload(d->source, envSourceFloats(d), s));
    CU(cudaEventRecord(c->evEnv[0], s));
    launchEnvBake(envBakeParams(d, d->sourceType == 0 ? nullptr : (keptSource ? c->envSource.ptr : fresh.ptr), c->envBakeScratch.ptr), levels, s);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->evEnv[1], s));
    envbake::ImportanceParams ip{};
    ip.cube = c->envBakeScratch.ptr; ip.faceSize = dim;
    { size_t off = 0; for (uint32_t m = 0; m < envbake::kImportanceMips; m++) { ip.mips[m] = c->envImportanceScratch.ptr + off; off += size_t(envbake::kImportanceDim >> m) * (envbake::kImportanceDim >> m) * 4; } }
    launchEnvImportance(ip, s);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->evEnv[2], s));
    // the cube: a new array only when its size changes (the old one stays in place until the update succeeds), otherwise the bake is copied over the one the kernels sample
    DeviceTexture grown;
    const bool newCube = !c->envCube.array || c->envFaceSize != dim || c->envMipLevels != levels;
    if (newCube) { rc = allocEnvCube(dim, levels, grown); if (rc != RTXPT_OK) return rc; }
    {
        size_t off = 0;
        for (uint32_t m = 0; m < levels; m++)
        {   // MIP m of the bake is already six faces back to back: one copy into the six layers
            const uint32_t n = dim >> m;
            cudaArray_t level; CU(cudaGetMipmappedArrayLevel(&level, newCube ? grown.array : c->envCube.array, m));
            cudaMemcpy3DParms cp{};
            cp.srcPtr = make_cudaPitchedPtr(c->envBakeScratch.ptr + off, size_t(n) * 16, n, n); cp.dstArray = level; cp.extent = make_cudaExtent(n, n, 6); cp.kind = cudaMemcpyDeviceToDevice;
            CU(cudaMemcpy3DAsync(&cp, s));
            off += size_t(6) * n * n * 4;
        }
    }
    CU(cudaEventRecord(c->evEnv[3], s));
    // hand-off to the host light bake: the importance chain (the quad-tree, lookup map, weights and proxy table stay LightBaker's)
    std::vector<std::vector<float>> chain(envbake::kImportanceMips);
    { size_t off = 0; for (uint32_t m = 0; m < envbake::kImportanceMips; m++) { chain[m].resize(size_t(envbake::kImportanceDim >> m) * (envbake::kImportanceDim >> m) * 4); CU(cudaMemcpyAsync(chain[m].data(), c->envImportanceScratch.ptr + off, chain[m].size() * 4, cudaMemcpyDeviceToHost, s)); off += chain[m].size(); } }
    CU(cudaStreamSynchronize(s));
    if (newCube) { c->envCube = std::move(grown); c->envFaceSize = dim; c->envMipLevels = levels; }
    if (fresh.ptr) { c->envSource = std::move(fresh); c->envSourceType = d->sourceType; c->envSourceWidth = d->sourceWidth; c->envSourceHeight = d->sourceType == 1 ? d->sourceHeight : d->sourceWidth; }
    LightBakeState& st = c->lightState;
    st.hasEnvCube = true; st.envMipCount = envbake::kImportanceMips; st.envRadianceMips = std::move(chain);
    c->lightsDirty = true;
    if (c->haveConstants) { rc = uploadLights(c); if (rc != RTXPT_OK) return rc; }
    CU(cudaEventRecord(c->evEnv[4], s)); CU(cudaEventSynchronize(c->evEnv[4]));
    for (int k = 0; k < 4; k++) CU(cudaEventElapsedTime(&c->envUpdateMs[k], c->evEnv[k], c->evEnv[k + 1]));
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_last_env_update_ms(rtxpt_ctx* c, float* outMs4)
{
    if (!c || !outMs4) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    memcpy(outMs4, c->envUpdateMs, sizeof(c->envUpdateMs));
    return RTXPT_OK;
}

// ---- NEE-AT temporal feedback (SURVEY §8f row 1) ------------------------------------------------------------------------------------------------------------------
// Frame order (Sample.cpp:1412, :2438-2520): set_constants; neeat_update_begin; [realtime: BUILD pass]; neeat_update_end; radiance pass(es).  rtxpt_b200_path_trace_realtime runs
// update_end itself after its BUILD pass; reference mode calls it explicitly (depth / motion guides of the previous frame, as RTXPT's render targets hold at that point).
static bool neeatActive(const rtxpt_ctx* c) { return c->haveConstants && c->consts.NEEType == 2 && c->consts.NEEATFeedback != 0; }
static int neeatEnsure(rtxpt_ctx* c, cudaStream_t s)
{
    rtxpt_ctx::Neeat& n = c->na;
    const uint32_t W = c->tableWidth, H = c->tableHeight, L = uint32_t(c->lightState.lights.size());
    if (n.allocated && n.host.W == W && n.host.H == H && n.lightCount == L) return RTXPT_OK;
    if (n.allocated && n.host.W == W && n.host.H == H && L <= n.lightCapacity) { n.lightCount = L; return RTXPT_OK; }       // the light list changed length: per-light arrays have headroom, the feedback state stays
    CU(syncContext(c)); CU(cudaStreamSynchronize(s));
    n = rtxpt_ctx::Neeat(); n.host.reset(W, H); n.lightCount = L;
    const size_t P = size_t(W) * H, B = size_t((W + 1) / 2) * ((H + 1) / 2), T = size_t(neeat::HostState::tilesX(W)) * neeat::HostState::tilesY(H) * neeat::kLocalProxyCount;
    const uint32_t Lcap = L + 4096u; n.lightCapacity = Lcap;        // headroom for lights added later (rtxpt_b200_update_lights); beyond it the feedback state starts over
    const size_t proxyCapacity = size_t(neeat::kProxyRatio) * std::max<uint32_t>(Lcap, neeat::kMaxLights / 10) + Lcap;           // every light rounds its share up
    CU(n.fbWeight.alloc(P)); CU(n.scratchWeight.alloc(P)); CU(n.blendedWeight.alloc(B)); CU(n.historyDepth.alloc(P)); CU(n.fbCandidate.alloc(P)); CU(n.scratchCandidate.alloc(P)); CU(n.blendedCandidate.alloc(B));
    CU(n.local.alloc(T)); CU(n.counters.alloc(size_t(Lcap) + 1)); CU(n.proxyCounters.alloc(Lcap)); CU(n.proxyOffsets.alloc(size_t(Lcap) + 1)); CU(n.proxyIndices.alloc(proxyCapacity)); CU(n.samplingProxyCount.alloc(1));
    CU(n.scanBlockSums.alloc(1024)); CU(n.lightWeights.alloc(Lcap)); CU(n.rrFix.alloc(c->capacity)); CU(n.shadowFeedback.alloc(c->capacity));
    CU(n.pastToCurrent.alloc(Lcap)); CU(n.currentToPast.alloc(Lcap));
    CU(n.rrFix.fill(0, s));
    CU(n.weights[0].alloc(Lcap)); CU(n.weights[1].alloc(Lcap)); CU(n.weightGroupSums.alloc((Lcap + 4095) / 4096 + 1)); CU(n.weightsSum.alloc(1));
    CU(n.weights[0].fill(0, s)); CU(n.weights[1].fill(0, s));
    CU(n.fbWeight.fill(0, s)); CU(n.scratchWeight.fill(0, s)); CU(n.blendedWeight.fill(0, s)); CU(n.historyDepth.fill(0, s));
    CU(n.fbCandidate.fill(0xFF, s)); CU(n.scratchCandidate.fill(0xFF, s)); CU(n.blendedCandidate.fill(0xFF, s));
    CU(n.local.fill(0, s)); CU(n.samplingProxyCount.fill(0, s));
    n.allocated = true;
    return RTXPT_OK;
}
static void neeatBind(rtxpt_ctx* c)
{
    rtxpt_ctx::Neeat& n = c->na; neeat::Params& p = n.params;
    p.fbWeight = n.fbWeight.ptr; p.fbCandidate = n.fbCandidate.ptr; p.scratchWeight = n.scratchWeight.ptr; p.scratchCandidate = n.scratchCandidate.ptr; p.blendedWeight = n.blendedWeight.ptr;
    p.blendedCandidate = n.blendedCandidate.ptr; p.historyDepth = n.historyDepth.ptr; p.localSamplingBuffer = n.local.ptr; p.feedbackCounters = n.counters.ptr; p.lightWeights = n.lightWeights.ptr;
    p.proxyCounters = n.proxyCounters.ptr; p.proxyOffsets = n.proxyOffsets.ptr; p.proxyIndices = n.proxyIndices.ptr; p.samplingProxyCount = n.samplingProxyCount.ptr;
    p.depth = c->depth.ptr; p.motion = c->motionVectors.ptr;
    p.lightRecords = reinterpret_cast<const uint4*>(c->dLights.ptr); p.curWeights = n.weights[n.weightPingPong].ptr; p.histWeights = n.weights[n.weightPingPong ^ 1u].ptr;
    p.weightGroupSums = n.weightGroupSums.ptr; p.weightsSumDev = n.weightsSum.ptr;
    p.pastToCurrent = n.remapActive ? n.pastToCurrent.ptr : nullptr; p.currentToPast = n.remapActive ? n.currentToPast.ptr : nullptr;
}
// ---- dynamic analytic lights: Donut's scene lights move, dim, appear and disappear between frames; RTXPT re-bakes its light list every frame (LightsBaker::UpdateBegin) ----------
extern "C" RTXPT_API int rtxpt_b200_update_lights(rtxpt_ctx* c, const RtxptLightDesc* lights, uint32_t count)
{
    if (!c || (count && !lights)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    LightBakeState& st = c->lightState;
    if (size_t(kEnvQuadLightCount) + count + st.triangleLights.size() >= kMaxLights) return fail(RTXPT_ERR_INVALID_ARGUMENT, "too many lights (%u analytic + %zu emissive triangles)", count, st.triangleLights.size());
    for (const RtxptSubInstanceData& si : c->hSubInstances)
        if (si.AnalyticProxyLightIndex != 0xFFFFFFFFu && si.AnalyticProxyLightIndex - kEnvQuadLightCount >= count) return fail(RTXPT_ERR_INVALID_ARGUMENT, "proxy geometry stands in for light %u, %u lights given", si.AnalyticProxyLightIndex - kEnvQuadLightCount, count);
    cudaSetDevice(c->device);
    CU(syncContext(c));
    const int64_t delta = int64_t(count) - int64_t(st.analyticLights.size());
    LightBaker::setAnalyticLights(lights, count, st);
    if (delta != 0)
    {   // the emissive triangles sit behind the analytic lights: their block offsets move with the count
        for (RtxptSubInstanceData& si : c->hSubInstances) if (si.EmissiveLightMappingOffset != 0xFFFFFFFFu) si.EmissiveLightMappingOffset = uint32_t(int64_t(si.EmissiveLightMappingOffset) + delta);
        CU(cudaMemcpy(c->dSubInstances.ptr, c->hSubInstances.data(), c->hSubInstances.size() * sizeof(RtxptSubInstanceData), cudaMemcpyHostToDevice));
    }
    c->lightsDirty = true;
    if (c->haveConstants) return uploadLights(c);
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_neeat_reset(rtxpt_ctx* c)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    c->na = rtxpt_ctx::Neeat();
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_neeat_update_begin(rtxpt_ctx* c, void* cudaStream)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    if (!c->haveScene || !neeatActive(c)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEE-AT feedback needs a scene and constants with NEEType == 2 and NEEATFeedback != 0");
    if (c->lightState.proxyIndices.empty()) return fail(RTXPT_ERR_INVALID_ARGUMENT, "the scene has no lights to sample");
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    int rc = neeatEnsure(c, s); if (rc != RTXPT_OK) return rc;
    rtxpt_ctx::Neeat& n = c->na;
    // the power-based weights follow the light list (uploadLights re-bakes them when the environment or the importance settings change)
    CU(cudaMemcpyAsync(n.lightWeights.ptr, c->lightState.weights.data(), size_t(n.lightCount) * 4, cudaMemcpyHostToDevice, s));
    // dynamic light list: the feedback of last frame names lights by their index in last frame's list (LightsBaker.cpp:1086-1225)
    n.remapActive = false;
    if (n.snap.valid && n.snapVersion != c->lightVersion && n.host.feedbackBufferFilled)
    {
        LightBaker::buildRemap(n.snap, c->lightState, n.hPastToCurrent, n.hCurrentToPast);
        if (n.hPastToCurrent.size() > n.pastToCurrent.count || n.hCurrentToPast.size() > n.currentToPast.count) return fail(RTXPT_ERR_INVALID_ARGUMENT, "light list outgrew the feedback state");
        CU(cudaMemcpyAsync(n.pastToCurrent.ptr, n.hPastToCurrent.data(), n.hPastToCurrent.size() * 4, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(n.currentToPast.ptr, n.hCurrentToPast.data(), n.hCurrentToPast.size() * 4, cudaMemcpyHostToDevice, s));
        n.remapActive = true;
    }
    if (!n.snap.valid || n.snapVersion != c->lightVersion) { LightBaker::snapshot(c->lightState, n.snap); n.snapVersion = c->lightVersion; }
    neeat::beginFrame(n.host, n.params, c->consts.NEEType, n.lightCount, c->lightState.weightsSum, c->consts.NEEATImportanceBoost, c->haveView ? c->worldToClip : nullptr);
    n.weightPingPong ^= 1u;                 // last frame's boosted weights become the historic ones
    neeatBind(c);
    launchNeeatUpdateBegin(n.params, n.host.settings.preFilter, n.scanBlockSums.ptr, c->grid.smCount, s);
    CU(cudaGetLastError());
    n.frameBegun = true; n.frameEnded = false;
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_neeat_update_end(rtxpt_ctx* c, void* cudaStream)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    if (!neeatActive(c) || !c->na.allocated || !c->na.frameBegun) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_neeat_update_begin has not run for this frame");
    if (!c->depth.ptr || !c->motionVectors.ptr) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEE-AT feedback reprojects with the depth / motion guides: create the context with RTXPT_CFG_EXPORT_GUIDES or use realtime mode");
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    neeatBind(c);
    launchNeeatUpdateEnd(c->na.params, s);
    CU(cudaGetLastError());
    neeat::endFrame(c->na.host, c->na.params);
    c->na.frameBegun = false; c->na.frameEnded = true;
    return RTXPT_OK;
}
// debugging / tests: `what` as in the oracle's oracle_neeat_get (0-1 feedback, 2-3 processed, 4-5 blended reservoirs, 6 tile lists, 7 proxy counters, 8 control words, 11 proxy table)
extern "C" RTXPT_API int rtxpt_b200_neeat_readback(rtxpt_ctx* c, int what, void* dst, size_t dstBytes, size_t* outBytes)
{
    if (!c || !dst || !outBytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->na.allocated) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEE-AT feedback state does not exist before rtxpt_b200_neeat_update_begin");
    cudaSetDevice(c->device);
    rtxpt_ctx::Neeat& n = c->na; const neeat::Params& p = n.params;
    CU(syncContext(c));
    uint32_t total = 0; CU(cudaMemcpy(&total, n.samplingProxyCount.ptr, 4, cudaMemcpyDeviceToHost));
    const void* src = nullptr; size_t bytes = 0; uint32_t ctl[8];
    const size_t P = size_t(p.W) * p.H, B = size_t(p.blendedW) * p.blendedH;
    switch (what)
    {
    case 0: src = n.fbWeight.ptr; bytes = P * 4; break;          case 1: src = n.fbCandidate.ptr; bytes = P * 4; break;
    case 2: src = n.scratchWeight.ptr; bytes = P * 4; break;     case 3: src = n.scratchCandidate.ptr; bytes = P * 4; break;
    case 4: src = n.blendedWeight.ptr; bytes = B * 4; break;     case 5: src = n.blendedCandidate.ptr; bytes = B * 4; break;
    case 6: src = n.local.ptr; bytes = n.local.count * 4; break; case 7: src = n.proxyCounters.ptr; bytes = size_t(n.lightCount) * 4; break;
    case 11: src = n.proxyIndices.ptr; bytes = size_t(total) * 4; break;
    case 8:
    {
        uint32_t invalid = 0; CU(cudaMemcpy(&invalid, n.counters.ptr + n.lightCount, 4, cudaMemcpyDeviceToHost));
        ctl[0] = p.tilesX; ctl[1] = p.tilesY; ctl[2] = p.jitterX; ctl[3] = p.jitterY; ctl[4] = total; ctl[5] = p.updateCounter; ctl[6] = p.lastFrameFeedbackAvailable;
        ctl[7] = p.lastFrameFeedbackAvailable ? p.W * p.H - invalid : 0u;
        if (dstBytes < sizeof(ctl)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "destination too small"); memcpy(dst, ctl, sizeof(ctl)); *outBytes = sizeof(ctl); return RTXPT_OK;
    }
    default: return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown NEE-AT buffer %d", what);
    }
    if (dstBytes < bytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "destination too small (%zu < %zu)", dstBytes, bytes);
    CU(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    *outBytes = bytes;
    return RTXPT_OK;
}
// tests: overwrite the feedback reservoirs (f32 weight, u32 candidate, image sized) and mark them as filled
extern "C" RTXPT_API int rtxpt_b200_neeat_debug_set_feedback(rtxpt_ctx* c, const float* weight, const uint32_t* candidate)
{
    if (!c || !weight || !candidate) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->na.allocated) return fail(RTXPT_ERR_INVALID_ARGUMENT, "NEE-AT feedback state does not exist before rtxpt_b200_neeat_update_begin");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    const size_t P = size_t(c->na.host.W) * c->na.host.H;
    CU(cudaMemcpy(c->na.fbWeight.ptr, weight, P * 4, cudaMemcpyHostToDevice)); CU(cudaMemcpy(c->na.fbCandidate.ptr, candidate, P * 4, cudaMemcpyHostToDevice));
    c->na.host.feedbackBufferFilled = true;
    return RTXPT_OK;
}

// ---- ReBLUR (NRD) for one stable plane ------------------------------------------------------------------------------------------------------------------
// settings and per-frame constants: reblur_host.h
static int ensureReblurPools(rtxpt_ctx* c, cudaStream_t s)
{
    if (c->reblurWidth == c->tableWidth && c->reblurHeight == c->tableHeight) return RTXPT_OK;
    CU(syncContext(c)); CU(cudaStreamSynchronize(s));
    const size_t P = size_t(c->tableWidth) * c->tableHeight, T = size_t((c->tableWidth + 15) / 16) * ((c->tableHeight + 15) / 16);
    for (auto& h : c->reblur)
    {
        CU(h.prevViewZ.alloc(P)); CU(h.prevNormalRoughness.alloc(P)); CU(h.prevInternalData.alloc(P)); CU(h.diffFast.alloc(P)); CU(h.specFast.alloc(P)); CU(h.diffHistory.alloc(P)); CU(h.specHistory.alloc(P));
        CU(h.prevViewZ.fill(0, s)); CU(h.prevNormalRoughness.fill(0, s)); CU(h.prevInternalData.fill(0, s)); CU(h.diffFast.fill(0, s)); CU(h.specFast.fill(0, s)); CU(h.diffHistory.fill(0, s)); CU(h.specHistory.fill(0, s));
        for (int i = 0; i < 2; i++)
        {
            CU(h.tracking[i].alloc(P)); CU(h.diffLuma[i].alloc(P)); CU(h.specLuma[i].alloc(P));
            CU(h.tracking[i].fill(0, s)); CU(h.diffLuma[i].fill(0, s)); CU(h.specLuma[i].fill(0, s));
        }
        h.valid = false; h.pingPong = 0;
    }
    CU(c->rbTiles.alloc(T)); CU(c->rbTmp1Diff.alloc(P)); CU(c->rbTmp1Spec.alloc(P)); CU(c->rbTmp2Diff.alloc(P)); CU(c->rbTmp2Spec.alloc(P)); CU(c->rbOutDiff.alloc(P)); CU(c->rbOutSpec.alloc(P));
    CU(c->rbTrackingT.alloc(P)); CU(c->rbDiffFastT.alloc(P)); CU(c->rbSpecFastT.alloc(P)); CU(c->rbData1.alloc(P)); CU(c->rbData2.alloc(P));
    CU(c->rbTmp1Diff.fill(0, s)); CU(c->rbTmp1Spec.fill(0, s)); CU(c->rbTmp2Diff.fill(0, s)); CU(c->rbTmp2Spec.fill(0, s)); CU(c->rbOutDiff.fill(0, s)); CU(c->rbOutSpec.fill(0, s));
    CU(c->rbTrackingT.fill(0, s)); CU(c->rbDiffFastT.fill(0, s)); CU(c->rbSpecFastT.fill(0, s)); CU(c->rbData1.fill(0, s)); CU(c->rbData2.fill(0, s));
    c->reblurWidth = c->tableWidth; c->reblurHeight = c->tableHeight;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_reblur_denoise(rtxpt_ctx* c, uint32_t stablePlaneIndex, const RtxptReblurFrame* f, void* cudaStream)
{
    if (!c || !f) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (stablePlaneIndex >= RTXPT_STABLE_PLANE_COUNT) return fail(RTXPT_ERR_INVALID_ARGUMENT, "bad plane index");
    if (c->denoiserWidth != c->tableWidth || c->denoiserHeight != c->tableHeight || c->denoiserWidth == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_denoiser_prepare_inputs has not run: ReBLUR reads RTXPT_BUFFER_DENOISER_*");
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    int rc = ensureReblurPools(c, s); if (rc != RTXPT_OK) return rc;
    rtxpt_ctx::ReblurHistory& h = c->reblur[stablePlaneIndex];
    const uint32_t W = c->tableWidth, H = c->tableHeight;
    const RtxptReblurSettings& settings = c->reblurSettings;
    rb::Params p{}; rb::fillFrameParams(p, W, H, f, h.valid, settings);
    // resources; without the disocclusion-threshold mix (isDisocclusionThresholdMixAvailable false) TemporalAccumulation reads a mix of 0
    p.viewZ = c->dnViewZ.ptr; p.normalRoughness = c->dnNormalRoughness.ptr; p.motion = f->ignoreMotionVectors ? nullptr : c->dnMotion.ptr;
    p.disocclusionMix = settings.useAlternateDisocclusionThresholdMix ? c->dnDisocclusionMix.ptr : nullptr; p.inDiff = c->dnDiff.ptr; p.inSpec = c->dnSpec.ptr;
    p.tiles = c->rbTiles.ptr; p.tmp1Diff = c->rbTmp1Diff.ptr; p.tmp1Spec = c->rbTmp1Spec.ptr; p.tmp2Diff = c->rbTmp2Diff.ptr; p.tmp2Spec = c->rbTmp2Spec.ptr;
    p.trackingTransient = c->rbTrackingT.ptr; p.diffFastTransient = c->rbDiffFastT.ptr; p.specFastTransient = c->rbSpecFastT.ptr; p.data1 = c->rbData1.ptr; p.data2 = c->rbData2.ptr;
    p.prevViewZ = h.prevViewZ.ptr; p.prevNormalRoughness = h.prevNormalRoughness.ptr; p.prevInternalData = h.prevInternalData.ptr; p.diffHistory = h.diffHistory.ptr; p.specHistory = h.specHistory.ptr;
    p.diffFast = h.diffFast.ptr; p.specFast = h.specFast.ptr;
    const uint32_t prev = h.pingPong, curr = prev ^ 1u;
    p.trackingPrev = h.tracking[prev].ptr; p.trackingCurr = h.tracking[curr].ptr; p.diffLumaPrev = h.diffLuma[prev].ptr; p.diffLumaCurr = h.diffLuma[curr].ptr; p.specLumaPrev = h.specLuma[prev].ptr; p.specLumaCurr = h.specLuma[curr].ptr;
    p.outDiff = c->rbOutDiff.ptr; p.outSpec = c->rbOutSpec.ptr;
    launchReblurFrame(p, settings.hitDistanceReconstructionMode, !(c->cfg.flags & RTXPT_CFG_REBLUR_UNTILED), s);
    CU(cudaGetLastError());
    h.pingPong = curr; h.valid = true;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_default_reblur_settings(RtxptReblurSettings* out)
{
    if (!out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    *out = rb::defaultSettings();
    return RTXPT_OK;
}
// m_ui.ReblurSettings -> nrd::SetDenoiserSettings (NrdIntegration.cpp:364-368): taken from the next frame on, history kept
extern "C" RTXPT_API int rtxpt_b200_set_reblur_settings(rtxpt_ctx* c, const RtxptReblurSettings* settings)
{
    if (!c || !settings) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (const char* why = rb::settingsError(*settings)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "ReBLUR settings refused: %s", why);
    c->reblurSettings = *settings;
    return RTXPT_OK;
}

// Sample::Denoise (Rtxpt/Sample.cpp:2560-2618): for plane = active - 1 .. 0 { prepare inputs (the first one also seeds the output with the stable radiance); NRD; final merge }
extern "C" RTXPT_API int rtxpt_b200_denoise_realtime(rtxpt_ctx* c, const RtxptDenoiserConstants* k, const RtxptReblurFrame* f, void* cudaStream)
{
    int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
    if (!k || !f) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null constants");
    cudaStream_t s = pickStream(c, cudaStream);
    if (!c->evDnStop) { CU(c->evDnStart.create(cudaEventCreateWithFlags, cudaEventDefault)); CU(c->evDnStop.create(cudaEventCreateWithFlags, cudaEventDefault)); }
    CU(cudaEventRecord(c->evDnStart, s));
    rc = rtxpt_b200_denoise_spec_hit_t(c, cudaStream); if (rc != RTXPT_OK) return rc;          // "Denoising Guides Bake" precedes Sample::Denoise in the frame
    bool first = true;
    for (int plane = int(c->realtime.activeStablePlaneCount) - 1; plane >= 0; plane--)
    {
        rc = rtxpt_b200_denoiser_prepare_inputs(c, uint32_t(plane), first ? 1 : 0, k, cudaStream); if (rc != RTXPT_OK) return rc;
        rc = rtxpt_b200_reblur_denoise(c, uint32_t(plane), f, cudaStream); if (rc != RTXPT_OK) return rc;
        rc = rtxpt_b200_denoiser_final_merge(c, uint32_t(plane), nullptr, nullptr, cudaStream); if (rc != RTXPT_OK) return rc;
        first = false;
    }
    CU(cudaEventRecord(c->evDnStop, s)); c->denoiseTimed = true;
    return RTXPT_OK;
}
// device time of the last rtxpt_b200_denoise_realtime call (CUDA events on its stream); waits for it to finish
extern "C" RTXPT_API int rtxpt_b200_last_denoise_ms(rtxpt_ctx* c, float* outMs)
{
    if (!c || !outMs) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->denoiseTimed) return fail(RTXPT_ERR_INVALID_ARGUMENT, "rtxpt_b200_denoise_realtime has not run");
    cudaSetDevice(c->device);
    CU(cudaEventSynchronize(c->evDnStop));
    CU(cudaEventElapsedTime(outMs, c->evDnStart, c->evDnStop));
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_reset_accumulation(rtxpt_ctx* c)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    c->accumulatedSamples = 0;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_synchronize(rtxpt_ctx* c)
{
    if (!c) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null context");
    cudaSetDevice(c->device);
    CU(syncContext(c));
    return RTXPT_OK;
}

static int targetInfo(rtxpt_ctx* c, int buffer, void** ptr, size_t* bytes)
{
    const size_t P = size_t(c->tableWidth) * c->tableHeight;
    switch (buffer)
    {
    case RTXPT_BUFFER_OUTPUT_COLOR_F16: *ptr = c->outputColor.ptr; *bytes = P * 8; return RTXPT_OK;
    case RTXPT_BUFFER_ACCUMULATED_F32: *ptr = c->accumulated.ptr; *bytes = P * 16; return RTXPT_OK;
    case RTXPT_BUFFER_DEPTH_F32: *ptr = c->depth.ptr; *bytes = P * 4; return RTXPT_OK;
    case RTXPT_BUFFER_MOTION_VECTORS_F16: *ptr = c->motionVectors.ptr; *bytes = P * 8; return RTXPT_OK;
    case RTXPT_BUFFER_THROUGHPUT_R11G11B10: *ptr = c->throughput.ptr; *bytes = P * 4; return RTXPT_OK;
    case RTXPT_BUFFER_STABLE_PLANES: case RTXPT_BUFFER_STABLE_PLANES_HEADER: case RTXPT_BUFFER_STABLE_RADIANCE_F16: case RTXPT_BUFFER_SPECULAR_HITT_F32:
        if (!c->haveRealtime || c->realtimeWidth != c->tableWidth || c->realtimeHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "realtime buffers do not exist before rtxpt_b200_set_realtime");
        if (buffer == RTXPT_BUFFER_STABLE_PLANES) { *ptr = c->stablePlanes.ptr; *bytes = c->stablePlanes.count * sizeof(RtxptStablePlane); }
        else if (buffer == RTXPT_BUFFER_STABLE_PLANES_HEADER) { *ptr = c->stablePlanesHeader.ptr; *bytes = P * 16; }
        else if (buffer == RTXPT_BUFFER_STABLE_RADIANCE_F16) { *ptr = c->stableRadiance.ptr; *bytes = P * 8; }
        else { *ptr = c->specularHitT.ptr; *bytes = P * 4; }
        return RTXPT_OK;
    case RTXPT_BUFFER_DENOISER_VIEWSPACE_Z_F32: case RTXPT_BUFFER_DENOISER_MOTION_VECTORS_F16: case RTXPT_BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2: case RTXPT_BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16:
    case RTXPT_BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16: case RTXPT_BUFFER_DENOISER_DISOCCLUSION_MIX_R8: case RTXPT_BUFFER_COMBINED_HISTORY_CLAMP_RELAX_R8:
        if (c->denoiserWidth != c->tableWidth || c->denoiserHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "denoiser buffers do not exist before rtxpt_b200_denoiser_prepare_inputs");
        switch (buffer)
        {
        case RTXPT_BUFFER_DENOISER_VIEWSPACE_Z_F32: *ptr = c->dnViewZ.ptr; *bytes = P * 4; break;
        case RTXPT_BUFFER_DENOISER_MOTION_VECTORS_F16: *ptr = c->dnMotion.ptr; *bytes = P * 8; break;
        case RTXPT_BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2: *ptr = c->dnNormalRoughness.ptr; *bytes = P * 4; break;
        case RTXPT_BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16: *ptr = c->dnDiff.ptr; *bytes = P * 8; break;
        case RTXPT_BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16: *ptr = c->dnSpec.ptr; *bytes = P * 8; break;
        case RTXPT_BUFFER_DENOISER_DISOCCLUSION_MIX_R8: *ptr = c->dnDisocclusionMix.ptr; *bytes = P; break;
        default: *ptr = c->dnHistoryClampRelax.ptr; *bytes = P; break;
        }
        return RTXPT_OK;
    case RTXPT_BUFFER_DEBUG_VIZ_F16:
        if (c->debugViz.count != P) return fail(RTXPT_ERR_INVALID_ARGUMENT, "the debug view target does not exist before a path_trace call with a debug view set");
        *ptr = c->debugViz.ptr; *bytes = P * 8; return RTXPT_OK;
    case RTXPT_BUFFER_RR_DIFFUSE_ALBEDO_R11G11B10: case RTXPT_BUFFER_RR_SPECULAR_ALBEDO_R11G11B10: case RTXPT_BUFFER_RR_NORMALS_ROUGHNESS_F16: case RTXPT_BUFFER_RR_SPECULAR_MOTION_VECTORS_F16:
        if (c->rrWidth != c->tableWidth || c->rrHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "the DLSS-RR inputs do not exist before rtxpt_b200_dlss_rr_prepare_inputs");
        if (buffer == RTXPT_BUFFER_RR_DIFFUSE_ALBEDO_R11G11B10) { *ptr = c->rrDiffAlbedo.ptr; *bytes = P * 4; }
        else if (buffer == RTXPT_BUFFER_RR_SPECULAR_ALBEDO_R11G11B10) { *ptr = c->rrSpecAlbedo.ptr; *bytes = P * 4; }
        else if (buffer == RTXPT_BUFFER_RR_NORMALS_ROUGHNESS_F16) { *ptr = c->rrNormalsRoughness.ptr; *bytes = P * 8; }
        else { *ptr = c->rrSpecMotionVectors.ptr; *bytes = P * 4; }
        return RTXPT_OK;
    case RTXPT_BUFFER_LDR_COLOR_RGBA8:
        if (!c->toneMapped || c->ldrColor.count != P) return fail(RTXPT_ERR_INVALID_ARGUMENT, "the LDR colour does not exist before rtxpt_b200_tone_map");
        *ptr = c->ldrColor.ptr; *bytes = P * 4; return RTXPT_OK;
    case RTXPT_BUFFER_DENOISED_DIFF_RADIANCE_HITDIST_F16: case RTXPT_BUFFER_DENOISED_SPEC_RADIANCE_HITDIST_F16: case RTXPT_BUFFER_REBLUR_ACCUMULATED_FRAMES_RG8:
        if (c->reblurWidth != c->tableWidth || c->reblurHeight != c->tableHeight) return fail(RTXPT_ERR_INVALID_ARGUMENT, "ReBLUR buffers do not exist before rtxpt_b200_reblur_denoise");
        if (buffer == RTXPT_BUFFER_DENOISED_DIFF_RADIANCE_HITDIST_F16) { *ptr = c->rbOutDiff.ptr; *bytes = P * 8; }
        else if (buffer == RTXPT_BUFFER_DENOISED_SPEC_RADIANCE_HITDIST_F16) { *ptr = c->rbOutSpec.ptr; *bytes = P * 8; }
        else { *ptr = c->rbData1.ptr; *bytes = P * 2; }
        return RTXPT_OK;
    default: return fail(RTXPT_ERR_INVALID_ARGUMENT, "unknown buffer %d", buffer);
    }
}

extern "C" RTXPT_API int rtxpt_b200_device_ptr(rtxpt_ctx* c, int buffer, void** outPtr, size_t* outBytes)
{
    if (!c || !outPtr || !outBytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    return targetInfo(c, buffer, outPtr, outBytes);
}

extern "C" RTXPT_API int rtxpt_b200_readback(rtxpt_ctx* c, int buffer, void* dst, size_t dstBytes)
{
    if (!c || !dst) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    void* src; size_t bytes;
    int rc = targetInfo(c, buffer, &src, &bytes); if (rc != RTXPT_OK) return rc;
    if (dstBytes < bytes) return fail(RTXPT_ERR_INVALID_ARGUMENT, "destination too small (%zu < %zu)", dstBytes, bytes);
    CU(joinCallerStream(c));                // the frame may have been queued on the caller's stream: the copy on the context stream is ordered after it
    CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_render_frame(rtxpt_ctx* c, const RtxptPathTracerConstants* k, uint32_t firstSubSampleIndex, uint32_t subSampleCount, void* dst, size_t dstBytes)
{
    int rc = rtxpt_b200_set_constants(c, k); if (rc != RTXPT_OK) return rc;
    rc = rtxpt_b200_path_trace(c, firstSubSampleIndex, subSampleCount, 1, nullptr); if (rc != RTXPT_OK) return rc;
    return rtxpt_b200_readback(c, RTXPT_BUFFER_ACCUMULATED_F32, dst, dstBytes);
}

extern "C" RTXPT_API int rtxpt_b200_get_stats(rtxpt_ctx* c, RtxptStats* out)
{
    if (!c || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    memset(out, 0, sizeof(*out));
    CU(syncContext(c));
    out->bvhNodeCount = c->bvhNodeCount; out->bvhTriangleCount = c->bvhTriCount; out->bvhBuildSeconds = c->bvhBuildSeconds;
    out->lightCount = uint32_t(c->lightState.lights.size()); out->lightProxyCount = uint32_t(c->lightState.proxyIndices.size());
    out->accumulatedSamples = c->accumulatedSamples;
    if (c->statsPending)
    {
        float ms = 0; CU(cudaEventElapsedTime(&ms, c->evStart, c->evStop));
        out->msTotal = ms;
        // counters hold the LAST batch; scale ray counts to the whole call when it was split into equal batches
        const uint32_t perLaunch = std::max(1u, c->lastSubSamplesPerLaunch);        // 1 while NEE-AT feedback is active, cfg.maxSubSamplesPerLaunch otherwise
        const uint32_t batches = (c->lastSubSamples + perLaunch - 1) / perLaunch;
        const uint32_t lastBatch = c->lastSubSamples - (batches - 1) * perLaunch;
        const double scale = double(c->lastSubSamples) / double(lastBatch);
        uint64_t scatter = 0, shadow = 0, nodes = 0, tests = 0, snodes = 0, stests = 0;
        for (uint32_t it = 0; it < c->lastIterations; it++)
        {
            uint64_t raysThisIteration = 0;
            for (uint32_t l = 0; l < c->lastLanes; l++)        // the lanes of the last batch each counted their own wavefront
            {
                const uint32_t* k = c->hCounters + size_t(l) * kCounterWords + it * kCountersPerIter;
                scatter += k[kCtrRayCount]; shadow += k[kCtrShadowCount] + k[kCtrShadowShort]; nodes += k[kCtrNodeVisits]; tests += k[kCtrTriTests];
                snodes += k[kCtrShadowNodeVisits]; stests += k[kCtrShadowTriTests]; raysThisIteration += k[kCtrRayCount];
            }
            if (it < 16) out->raysPerBounce[it] = uint64_t(raysThisIteration * scale);
        }
        out->scatterRays = uint64_t(scatter * scale); out->shadowRays = uint64_t(shadow * scale);
        out->traversalNodeVisits = uint64_t(nodes * scale); out->traversalTriTests = uint64_t(tests * scale);
        out->shadowNodeVisits = uint64_t(snodes * scale); out->shadowTriTests = uint64_t(stests * scale);
        for (size_t e = 0; e + 1 < c->evUsed; e += 2)
        {
            float t = 0; CU(cudaEventElapsedTime(&t, c->evPool[e], c->evPool[e + 1]));
            switch (c->evKind[e / 2]) { case 0: out->msTraceClosest += t; break; case 1: out->msTraceShadow += t; break; case 2: out->msShade += t; break; default: out->msOther += t; }
        }
        out->paths = uint64_t(c->pixelCount) * c->lastSubSamples;
        out->kernelLaunches = c->lastLaunches;
    }
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_get_opacity_mask_stats(rtxpt_ctx* c, RtxptOpacityMaskStats* out)
{
    if (!c || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    out->triangles = c->opacityMaskTriangles; out->microTrianglesPerTriangle = om::kMicroTriangles; out->transparent = c->opacityMaskStates[om::kTransparent];
    out->opaque = c->opacityMaskStates[om::kOpaque]; out->unknown = c->opacityMaskStates[om::kUnknown]; out->bakeSeconds = c->opacityMaskBakeSeconds;
    return RTXPT_OK;
}

// ---- multi-GPU tile exchange --------------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API int rtxpt_b200_tile_layout(rtxpt_ctx* c, uint32_t* outOwned, uint32_t* outPadded)
{
    if (!c || !outOwned || !outPadded) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (c->tableWidth == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set");
    *outOwned = c->pixelCount; *outPadded = c->paddedPixelsPerRank;
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_pack_owned(rtxpt_ctx* c, void* dDst, void* cudaStream)
{
    if (!c || !dDst) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (c->tableWidth == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set");
    cudaSetDevice(c->device);
    launchPackOwned(c->accumulated.ptr, c->pixelOfSlot.ptr, c->pixelCount, c->paddedPixelsPerRank, c->tableWidth, (float4*)dDst, c->grid, pickStream(c, cudaStream));
    CU(cudaGetLastError());
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_unpack_all(rtxpt_ctx* c, const void* dSrcAll, void* cudaStream)
{
    if (!c || !dSrcAll) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (c->tableWidth == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set");
    cudaSetDevice(c->device);
    launchUnpackAll((const float4*)dSrcAll, c->allPixelTable.ptr, c->paddedPixelsPerRank * c->cfg.tileWorld, c->tableWidth, c->accumulated.ptr, c->grid, pickStream(c, cudaStream));
    CU(cudaGetLastError());
    return RTXPT_OK;
}

// ---- multi-GPU exchange of the realtime frame's per-pixel images (SURVEY §8e, config 3): guides, NRD inputs per plane, output colour ---------------------------------------------
static int buildExchangeSet(rtxpt_ctx* c, const int* buffers, uint32_t count, ExchangeSet& e)
{
    if (!c || !buffers || count == 0 || count > kExchangeMaxImages) return fail(RTXPT_ERR_INVALID_ARGUMENT, "1..%u buffers", kExchangeMaxImages);
    if (c->tableWidth == 0) return fail(RTXPT_ERR_INVALID_ARGUMENT, "constants not set");
    const size_t P = size_t(c->tableWidth) * c->tableHeight;
    memset(&e, 0, sizeof(e)); e.count = count; e.width = c->tableWidth;
    uint64_t off = 0;
    for (uint32_t k = 0; k < count; k++)
    {
        if (buffers[k] == RTXPT_BUFFER_STABLE_PLANE_NEIGHBOUR_GUIDES)
        {   // not an image: per plane the branch ID and the packed normal, gathered from the header layers and the plane records by their own kernels
            const int rc = checkRealtimeReady(c); if (rc != RTXPT_OK) return rc;
            e.image[k] = nullptr; e.bytesPerPixel[k] = 24; e.segmentOffset[k] = off; off += (uint64_t(c->paddedPixelsPerRank) * 24 + 15u) & ~uint64_t(15);
            continue;
        }
        if (buffers[k] == RTXPT_BUFFER_STABLE_PLANES || buffers[k] == RTXPT_BUFFER_STABLE_PLANES_HEADER) return fail(RTXPT_ERR_INVALID_ARGUMENT, "buffer %d is not a plain per-pixel image", buffers[k]);
        void* ptr; size_t bytes; const int rc = targetInfo(c, buffers[k], &ptr, &bytes); if (rc != RTXPT_OK) return rc;
        const size_t bpp = bytes / P;
        if (bytes != bpp * P || (bpp != 1 && bpp != 4 && bpp != 8 && bpp != 16)) return fail(RTXPT_ERR_INVALID_ARGUMENT, "buffer %d: %zu bytes per pixel cannot be exchanged", buffers[k], bpp);
        e.image[k] = ptr; e.bytesPerPixel[k] = uint32_t(bpp); e.segmentOffset[k] = off;
        off += (uint64_t(c->paddedPixelsPerRank) * bpp + 15u) & ~uint64_t(15);
    }
    e.bytesPerRank = off;
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_exchange_bytes(rtxpt_ctx* c, const int* buffers, uint32_t count, size_t* outBytesPerRank)
{
    if (!outBytesPerRank) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    ExchangeSet e; const int rc = buildExchangeSet(c, buffers, count, e); if (rc != RTXPT_OK) return rc;
    *outBytesPerRank = size_t(e.bytesPerRank);
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_exchange_pack(rtxpt_ctx* c, const int* buffers, uint32_t count, void* dDst, void* cudaStream)
{
    if (!dDst) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    ExchangeSet e; const int rc = buildExchangeSet(c, buffers, count, e); if (rc != RTXPT_OK) return rc;
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    launchExchangePack(e, c->pixelOfSlot.ptr, c->pixelCount, c->paddedPixelsPerRank, dDst, c->grid, s);
    for (uint32_t k = 0; k < e.count; k++)
        if (!e.image[k]) { LaunchParams p; fillParams(c, p); fillRealtimeParams(c, p); launchRtPackPlaneGuides(p, c->paddedPixelsPerRank, static_cast<uint8_t*>(dDst) + e.segmentOffset[k], c->grid, s); }
    CU(cudaGetLastError());
    return RTXPT_OK;
}
extern "C" RTXPT_API int rtxpt_b200_exchange_unpack(rtxpt_ctx* c, const int* buffers, uint32_t count, const void* dSrcAll, void* cudaStream)
{
    if (!dSrcAll) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    ExchangeSet e; const int rc = buildExchangeSet(c, buffers, count, e); if (rc != RTXPT_OK) return rc;
    if (c->cfg.tileWorld <= 1) return RTXPT_OK;
    cudaSetDevice(c->device);
    cudaStream_t s = pickStream(c, cudaStream);
    launchExchangeUnpack(e, c->allPixelTable.ptr, c->paddedPixelsPerRank, c->cfg.tileWorld, c->cfg.tileRank, dSrcAll, c->grid, s);
    for (uint32_t k = 0; k < e.count; k++)
        if (!e.image[k]) { LaunchParams p; fillParams(c, p); fillRealtimeParams(c, p); launchRtUnpackPlaneGuides(p, c->allPixelTable.ptr, c->paddedPixelsPerRank, c->cfg.tileWorld, c->cfg.tileRank, dSrcAll, size_t(e.segmentOffset[k]), size_t(e.bytesPerRank), c->grid, s); }
    CU(cudaGetLastError());
    return RTXPT_OK;
}

// ---- inspection hooks -------------------------------------------------------------------------------------------------------------------------
extern "C" RTXPT_API int rtxpt_b200_trace_rays_device(rtxpt_ctx* c, const void* dRays, uint32_t count, int anyHit, void* dHits, uint32_t repeat, float* outMs)
{
    if (!c || !c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    cudaSetDevice(c->device);
    if (c->counters.count == 0) CU(c->counters.alloc(size_t(kCounterWords) * rtxpt_ctx::kMaxLanes));
    LaunchParams p; fillParams(c, p);
    CU(cudaMemsetAsync(c->counters.ptr, 0, 8, c->stream));
    if (repeat == 0) repeat = 1;
    CU(cudaEventRecord(c->evStart, c->stream));
    for (uint32_t r = 0; r < repeat; r++)
        launchTraceRays(p, c->grid, (const RtxptRay*)dRays, count, anyHit != 0, (RtxptHit*)dHits, (r == 0) ? c->counters.ptr : nullptr, c->counters.ptr + 4, c->stream);
    CU(cudaEventRecord(c->evStop, c->stream));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(c->hCounters, c->counters.ptr, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(syncContext(c));
    float ms = 0; cudaEventElapsedTime(&ms, c->evStart, c->evStop);
    if (outMs) *outMs = ms / float(repeat);
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_trace_rays(rtxpt_ctx* c, const RtxptRay* rays, uint32_t count, int anyHit, RtxptHit* outHits)
{
    if (!c || !rays || !outHits) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    if (!c->haveScene) return fail(RTXPT_ERR_NO_SCENE, "no scene uploaded");
    cudaSetDevice(c->device);
    DeviceArray<RtxptRay> dRays; DeviceArray<RtxptHit> dHits;
    CU(dRays.upload(rays, count, c->stream)); CU(dHits.alloc(count));
    int rc = rtxpt_b200_trace_rays_device(c, dRays.ptr, count, anyHit, dHits.ptr, 1, nullptr); if (rc != RTXPT_OK) return rc;
    CU(cudaMemcpy(outHits, dHits.ptr, size_t(count) * sizeof(RtxptHit), cudaMemcpyDeviceToHost));
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_set_view(rtxpt_ctx* c, const RtxptViewConstants* view)
{
    if (!c || !view) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    memcpy(c->worldToClip, view->matWorldToClip, sizeof(c->worldToClip)); c->haveView = true;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_get_lights(rtxpt_ctx* c, void* outLightInfos, uint32_t* ioLightCount, uint32_t* outProxyCounters, uint32_t* outProxyIndices, uint32_t* ioProxyCount)
{
    int rc = checkReady(c); if (rc != RTXPT_OK) return rc;
    if (!ioLightCount || !ioProxyCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    const uint32_t n = uint32_t(c->lightState.lights.size()), m = uint32_t(c->lightState.proxyIndices.size());
    // read back from the device: what the kernels actually sample
    if (outLightInfos && *ioLightCount >= n) CU(cudaMemcpy(outLightInfos, c->dLights.ptr, size_t(n) * 32, cudaMemcpyDeviceToHost));
    if (outProxyCounters && *ioLightCount >= n) CU(cudaMemcpy(outProxyCounters, c->dProxyCounters.ptr, size_t(n) * 4, cudaMemcpyDeviceToHost));
    if (outProxyIndices && *ioProxyCount >= m && m) CU(cudaMemcpy(outProxyIndices, c->dProxyIndices.ptr, size_t(m) * 4, cudaMemcpyDeviceToHost));
    *ioLightCount = n; *ioProxyCount = m;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_get_lights_ex(rtxpt_ctx* c, void* outLightInfoEx, uint32_t* ioAnalyticLightCount)
{
    int rc = checkReady(c); if (rc != RTXPT_OK) return rc;
    if (!ioAnalyticLightCount) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    const uint32_t n = uint32_t(c->lightState.analyticLightsEx.size());
    if (outLightInfoEx && *ioAnalyticLightCount >= n && n) CU(cudaMemcpy(outLightInfoEx, c->dLightsEx.ptr, size_t(n) * 16, cudaMemcpyDeviceToHost));
    *ioAnalyticLightCount = n;
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_debug_bsdf(rtxpt_ctx* c, const float* in, uint32_t count, float* out)
{
    if (!c || !in || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    DeviceArray<float> dIn, dOut;
    CU(dIn.upload(in, size_t(count) * 36, c->stream)); CU(dOut.alloc(size_t(count) * 16));
    launchDebugBsdf(dIn.ptr, count, dOut.ptr, c->stream);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, dOut.ptr, size_t(count) * 16 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    CU(syncContext(c));
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_debug_rng(rtxpt_ctx* c, const uint32_t* in, uint32_t count, uint32_t* out)
{
    if (!c || !in || !out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    cudaSetDevice(c->device);
    DeviceArray<uint32_t> dIn, dOut;
    CU(dIn.upload(in, size_t(count) * 4, c->stream)); CU(dOut.alloc(size_t(count) * 8));
    launchDebugRng(dIn.ptr, count, dOut.ptr, c->stream);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(out, dOut.ptr, size_t(count) * 8 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU(syncContext(c));
    return RTXPT_OK;
}

extern "C" RTXPT_API int rtxpt_b200_debug_live_resources(uint64_t* out)
{
    if (!out) return fail(RTXPT_ERR_INVALID_ARGUMENT, "null argument");
    *out = g_liveResources.load();
    return RTXPT_OK;
}
