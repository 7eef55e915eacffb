// kernels.h — host-callable launchers of the wavefront kernels (kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include "wavefront.cuh"

namespace pt {

struct GridConfig
{
    int smCount = 1; int traceBlocksPerSM = 1; int shadeBlocksPerSM = 1;
    // optional L2 access-policy window for the traversal kernels (BVH nodes kept resident in the persisting L2 carve-out while path state streams through)
    const void* l2WindowBase = nullptr; size_t l2WindowBytes = 0; float l2WindowHitRatio = 1.0f;
};

cudaError_t configureKernels(int maxSmemOptin);
void launchGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
// wavefront traversal (kernels.cu): closest-hit or shadow rays; reference mode takes rays in state order, realtime mode through the slot queue;
// the NEE-AT shadow kinds also feed visible samples back to the pixel's reservoir; the Multi kinds (NEEFullSamples > 1) only mark visible samples in their NEE blocks,
// which launchNeeResolve then applies.  countSteps selects the step-counting kernel of Closest and Shadow.
enum class TraceKind { Closest, ClosestRealtime, Shadow, ShadowRealtime, ShadowNeeat, ShadowRealtimeNeeat, ShadowMulti, ShadowRealtimeMulti, Count };
void launchTrace(TraceKind kind, const LaunchParams& p, const GridConfig& g, bool countSteps, cudaStream_t s);
void launchNeeResolve(const LaunchParams& p, const GridConfig& g, bool realtime, cudaStream_t s);
void launchShade(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
// realtime mode (realtime_kernels.cu)
void launchRtBuildGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchRtFillGenerate(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchRtShade(const LaunchParams& p, const GridConfig& g, bool fill, cudaStream_t s);
void launchRtFillCommit(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchRtMerge(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchRtDebugViz(const LaunchParams& p, const GridConfig& g, cudaStream_t s);          // StablePlanesDebugViz after the FILL passes (rtxpt_b200_set_debug_view)
void launchDnPrepareInputs(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchDnFinalMerge(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
struct DlssRrTargets;
void launchDnPrepareDlssRr(const LaunchParams& p, const DlssRrTargets& rr, const GridConfig& g, cudaStream_t s);     // DENOISER_DLSS_RR (denoiser_iface.cuh)
void launchCommitAccumulate(const LaunchParams& p, const GridConfig& g, cudaStream_t s);
void launchTraceRays(const LaunchParams& p, const GridConfig& g, const RtxptRay* dRays, uint32_t count, bool anyHit, RtxptHit* dHits, uint32_t* dCounters, uint32_t* dCursor, cudaStream_t s);
void launchPackOwned(const float4* image, const uint32_t* pixelOfSlot, uint32_t pixelCount, uint32_t paddedCount, uint32_t width, float4* dst, const GridConfig& g, cudaStream_t s);
void launchUnpackAll(const float4* srcAll, const uint32_t* allPixelTable, uint32_t totalEntries, uint32_t width, float4* image, const GridConfig& g, cudaStream_t s);
void launchInitTables(cudaStream_t s);       // lookup tables of the shading unit (Sobol byte tables); once per context
void launchDebugBsdf(const float* dIn, uint32_t count, float* dOut, cudaStream_t s);
void launchDebugRng(const uint32_t* dIn, uint32_t count, uint32_t* dOut, cudaStream_t s);

void launchDnSpecHitT(const float* src, const float* depth, float* dst, int W, int H, cudaStream_t s);      // DenoisingGuidesBaker::DenoiseSpecHitT, one pass
void launchShadeNeeat(const LaunchParams& p, const GridConfig& g, cudaStream_t s);                 // reference-mode shade with NEE-AT feedback (shade_kernels.cu)
void launchRtShadeNeeat(const LaunchParams& p, const GridConfig& g, cudaStream_t s);               // FILL pass shade with NEE-AT feedback (realtime_kernels.cu)
namespace skin { struct Params; }
constexpr uint32_t kExchangeMaxImages = 8;
struct ExchangeSet { void* image[kExchangeMaxImages]; uint32_t bytesPerPixel[kExchangeMaxImages]; uint64_t segmentOffset[kExchangeMaxImages]; uint64_t bytesPerRank; uint32_t count, width; };
void launchExchangePack(const ExchangeSet& e, const uint32_t* pixelOfSlot, uint32_t pixelCount, uint32_t paddedCount, void* dst, const GridConfig& g, cudaStream_t s);                 // kernels.cu
void launchExchangeUnpack(const ExchangeSet& e, const uint32_t* allPixelTable, uint32_t paddedCount, uint32_t world, uint32_t skipRank, const void* srcAll, const GridConfig& g, cudaStream_t s);
void launchRtPackPlaneGuides(const LaunchParams& p, uint32_t paddedCount, void* dst, const GridConfig& g, cudaStream_t s);                                                  // realtime_kernels.cu
void launchRtUnpackPlaneGuides(const LaunchParams& p, const uint32_t* allPixelTable, uint32_t paddedCount, uint32_t world, uint32_t skipRank, const void* srcAll, size_t segmentOffset, size_t bytesPerRank, const GridConfig& g, cudaStream_t s);
void launchSkin(const skin::Params& p, cudaStream_t s);                 // skinning_kernels.cu
void launchSkinInitPrev(const skin::Params& p, cudaStream_t s);         // previous-position range of a newly registered skin := the shade records' current corners
namespace tonemap { struct Params; }
void launchToneMap(const tonemap::Params& p, const void* src, bool srcIsF32, uint32_t pixelCount, double* partials, float* avgLuminance, uint32_t* dst, cudaStream_t s);      // tonemap_kernels.cu
namespace refit { struct Params; }
void launchRefit(const refit::Params& p, const uint32_t* levelStart, uint32_t levelCount, int smCount, cudaStream_t s);      // refit_kernels.cu
namespace envbake { struct Params; struct ImportanceParams; }
void launchEnvBake(const envbake::Params& p, uint32_t mipLevels, cudaStream_t s);                  // envbake_kernels.cu: EnvMapBaker BaseLayerCS + MIPReduceCS
void launchEnvImportance(const envbake::ImportanceParams& p, cudaStream_t s);                      // envbake_kernels.cu: BuildMIPDescentImportanceMapCS + its 2x2 MIP chain
namespace neeat { struct Params; }
void launchNeeatUpdateBegin(const neeat::Params& p, bool preFilter, uint* scanBlockSums, int smCount, cudaStream_t s);     // neeat_kernels.cu
void launchNeeatUpdateEnd(const neeat::Params& p, cudaStream_t s);
namespace rb { struct Params; }
// reblur_kernels.cu: the ReBLUR passes of one stable plane that the settings select (rb::routeFrame: hit-distance reconstruction mode, pre-pass radii in p); tiled: HitDistReconstruction through shared memory
void launchReblurFrame(const rb::Params& p, uint32_t hitDistanceReconstructionMode, bool tiled, cudaStream_t s);

} // namespace pt
