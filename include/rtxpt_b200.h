/*
 * rtxpt_b200.h — C ABI of the CUDA-native (H100, sm_90a) wavefront path tracer that drops in for RTXPT's single
 * PathTrace dispatch.
 *
 * Every entry point below replaces one piece of the reference's host→GPU boundary for that path.  The
 * citations (file:line, relative to the RTXPT source tree) name the reference interface it stands in for.
 * Plain C: pointers and sizes only, caller owns host memory, the library owns device memory, one context per GPU,
 * calls on one context are serialised by the caller (the reference renders from a single thread,
 * Rtxpt/Sample.cpp:1891-2313).
 *
 * All entry points return RTXPT_OK (0) or a negative status; rtxpt_b200_last_error() gives the message.
 */
#ifndef RTXPT_B200_H_
#define RTXPT_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define RTXPT_API __declspec(dllexport)
#else
#define RTXPT_API __attribute__((visibility("default")))
#endif

/* ------------------------------------------------------------------------------------------------------------------
 * Status codes (the reference has no formal convention: bool returns + donut::log::error, SURVEY §8b)
 * ---------------------------------------------------------------------------------------------------------------- */
enum {
    RTXPT_OK                    =  0,
    RTXPT_ERR_INVALID_ARGUMENT  = -1,
    RTXPT_ERR_NO_DEVICE         = -2,   /* no CUDA device / driver: the library never falls back to the CPU */
    RTXPT_ERR_CUDA              = -3,
    RTXPT_ERR_OUT_OF_MEMORY     = -4,
    RTXPT_ERR_NO_SCENE          = -5,
    RTXPT_ERR_UNSUPPORTED       = -6,
    RTXPT_ERR_INTERNAL          = -7
};

/* ------------------------------------------------------------------------------------------------------------------
 * Scene tables.  Layouts are byte-identical to what the reference binds for the dispatch
 * (Rtxpt/Sample.cpp:2315-2427): t1 SubInstanceData[], t2 InstanceData[], t3 GeometryData[], t5 PTMaterialData[],
 * bindless ByteAddressBuffer[] (index + vertex) and Texture2D[].
 * ---------------------------------------------------------------------------------------------------------------- */

/* External/Donut/include/donut/shaders/bindless.h:28-46 (64 bytes) */
typedef struct RtxptGeometryData {
    uint32_t numIndices;
    uint32_t numVertices;
    int32_t  indexBufferIndex;
    uint32_t indexOffset;           /* bytes */
    int32_t  vertexBufferIndex;
    uint32_t positionOffset;        /* bytes; float3 per vertex (12 B) */
    uint32_t prevPositionOffset;    /* 0xFFFFFFFF when absent */
    uint32_t texCoord1Offset;       /* bytes; float2 per vertex (8 B); 0xFFFFFFFF when absent */
    uint32_t texCoord2Offset;
    uint32_t normalOffset;          /* bytes; RGB8 snorm packed in one u32 (4 B); 0xFFFFFFFF when absent */
    uint32_t tangentOffset;         /* bytes; RGBA8 snorm (4 B); 0xFFFFFFFF when absent */
    uint32_t curveRadiusOffset;
    uint32_t materialIndex;
    uint32_t pad0, pad1, pad2;
} RtxptGeometryData;

/* External/Donut/include/donut/shaders/bindless.h:54-70 (112 bytes); transforms are row-major float3x4 */
typedef struct RtxptInstanceData {
    uint32_t flags;
    uint32_t firstGeometryInstanceIndex;    /* index of this instance's first SubInstanceData */
    uint32_t firstGeometryIndex;            /* index of this instance's first GeometryData */
    uint32_t numGeometries;
    float    transform[12];
    float    prevTransform[12];
} RtxptInstanceData;

/* Rtxpt/Shaders/SubInstanceData.h:23-46 (32 bytes, SUBINSTANCEDATA_EXTENDED) */
typedef struct RtxptSubInstanceData {
    uint32_t FlagsAndAlphaInfo;                         /* [15:0] alpha texture index, bit16 alpha tested, bit17 exclude from NEE, [31:24] cutoff*255 */
    uint32_t GlobalGeometryIndex_PTMaterialDataIndex;   /* [31:16] geometry index, [15:0] material index */
    uint32_t EmissiveLightMappingOffset;                /* filled by the library's light bake; callers pass 0xFFFFFFFF */
    uint32_t AnalyticProxyLightIndex;                   /* index into RtxptSceneDesc.lights of the analytic light this geometry stands in for (material flag
                                                           EnableAsAnalyticLightProxy), 0xFFFFFFFF for none; the library rebases it into its light list */
    uint32_t IndexBufferIndex_VertexBufferIndex;
    uint32_t IndexOffset;
    uint32_t TexCoord1Offset;
    uint32_t padding0;
} RtxptSubInstanceData;

#define RTXPT_SUBINST_FLAG_ALPHA_TESTED     (1u << 16)
#define RTXPT_SUBINST_FLAG_EXCLUDE_FROM_NEE (1u << 17)

/* Rtxpt/Shaders/PathTracer/Materials/MaterialPT.h:23-80 (128 bytes) */
#define RTXPT_MATFLAG_UseSpecularGlossModel          0x00000001u
#define RTXPT_MATFLAG_UseMetalRoughOrSpecularTexture 0x00000004u
#define RTXPT_MATFLAG_UseBaseOrDiffuseTexture        0x00000008u
#define RTXPT_MATFLAG_UseEmissiveTexture             0x00000010u
#define RTXPT_MATFLAG_UseNormalTexture               0x00000020u
#define RTXPT_MATFLAG_UseTransmissionTexture         0x00000080u
#define RTXPT_MATFLAG_MetalnessInRedChannel          0x00000100u
#define RTXPT_MATFLAG_ThinSurface                    0x00000200u
#define RTXPT_MATFLAG_PSDExclude                     0x00000400u
#define RTXPT_MATFLAG_EnableAsAnalyticLightProxy     0x00000800u
#define RTXPT_MATFLAG_IgnoreMeshTangentSpace         (1u << 12)
#define RTXPT_MATFLAG_NestedPriorityShift            28

typedef struct RtxptMaterialData {
    float    BaseOrDiffuseColor[3];
    uint32_t Flags;
    float    SpecularColor[3];
    int32_t  _padding0;
    float    EmissiveColor[3];
    float    ShadowNoLFadeout;
    float    Opacity;
    float    Roughness;
    float    Metalness;
    float    NormalTextureScale;
    float    _padding1;
    float    AlphaCutoff;
    float    TransmissionFactor;
    uint32_t BaseOrDiffuseTextureIndex;         /* (baseLOD<<24)|(mipLevels<<16)|bindlessIndex, Materials/MaterialsBaker.cpp:487-509 */
    uint32_t MetalRoughOrSpecularTextureIndex;
    uint32_t EmissiveTextureIndex;
    uint32_t NormalTextureIndex;
    uint32_t OcclusionTextureIndex;
    uint32_t TransmissionTextureIndex;
    float    IoR;
    float    ThicknessFactor;
    float    DiffuseTransmissionFactor;
    float    VolumeAttenuationColor[3];
    float    VolumeAttenuationDistance;
} RtxptMaterialData;

/* One bindless ByteAddressBuffer (index or vertex data), t_BindlessBuffers[] in Rtxpt/Shaders/Bindings/SceneBindings.hlsli */
typedef struct RtxptBufferDesc {
    const void* data;
    uint64_t    sizeBytes;
} RtxptBufferDesc;

/* One bindless Texture2D.  Uncompressed only in this tier (block-compressed DDS is SURVEY §8f row 3). */
enum {
    RTXPT_FORMAT_RGBA8_UNORM = 0,
    RTXPT_FORMAT_RGBA8_SRGB  = 1,   /* sRGB-decoded on fetch, like the reference's per-slot sRGB views (Materials/MaterialsBaker.cpp:63-72) */
    RTXPT_FORMAT_RGBA32_FLOAT = 2,
    /* Block-compressed textures kept compressed in HBM and decoded by the texture units on fetch, as the reference does (its .dds assets go to D3D block-compressed formats through
     * Donut's DDSFile.cpp / TextureCache.cpp): mips[] hold the raw 4x4 blocks, rows of ceil(w/4) blocks, 8 (BC1) or 16 (BC2/3/7) bytes each.  4-8x less texture memory and traffic
     * than the RGBA8 expansion.  The *_SRGB variants decode sRGB -> linear on fetch (base colour / emissive slots, Materials/MaterialsBaker.cpp:63-72). */
    RTXPT_FORMAT_BC1_UNORM = 3, RTXPT_FORMAT_BC1_SRGB = 4, RTXPT_FORMAT_BC2_UNORM = 5, RTXPT_FORMAT_BC2_SRGB = 6,
    RTXPT_FORMAT_BC3_UNORM = 7, RTXPT_FORMAT_BC3_SRGB = 8, RTXPT_FORMAT_BC7_UNORM = 9, RTXPT_FORMAT_BC7_SRGB = 10
};
#define RTXPT_MAX_MIPS 16
typedef struct RtxptTextureDesc {
    uint32_t    width, height;
    uint32_t    mipLevels;              /* full or partial chain, mip i is max(1,w>>i) x max(1,h>>i) */
    uint32_t    format;
    const void* mips[RTXPT_MAX_MIPS];   /* tightly packed rows */
} RtxptTextureDesc;

/* Environment cube (t10, Rtxpt/Shaders/Bindings/LightingBindings.hlsli; produced by Lighting/Distant/EnvMapBaker in
 * the reference).  Faces in D3D order +X,-X,+Y,-Y,+Z,-Z, RGBA32F, square, with a mip chain. */
typedef struct RtxptEnvCubeDesc {
    uint32_t     faceSize;              /* 0 = no environment map */
    uint32_t     mipLevels;
    const float* faces[6][RTXPT_MAX_MIPS];
} RtxptEnvCubeDesc;

/* Analytic scene lights: the fields of Donut's PointLight / SpotLight (+ RTXPT's radius extension, Rtxpt/ExtendedScene.h) that
 * LightsBaker's ConvertLight reads (Rtxpt/Lighting/LightsBaker.cpp:456-556).  A light with radius > 0 becomes a sphere light
 * (a spot: a sphere light with cone shaping); radius == 0 becomes a kPoint record, which the reference's shaders compile out
 * (POLYLIGHT_POINT_ENABLE 0, PolymorphicLightPTConfig.h:18) - it occupies a slot in the light list and is never sampled.
 * Directional lights are baked into the environment map by the reference (out of scope here). */
#define RTXPT_LIGHT_POINT 1u
#define RTXPT_LIGHT_SPOT  2u
typedef struct RtxptLightDesc {
    uint32_t type;              /* RTXPT_LIGHT_* */
    float    position[3];
    float    direction[3];      /* spot axis (need not be normalised) */
    float    color[3];
    float    intensity;
    float    radius;
    float    innerAngle;        /* degrees (spot) */
    float    outerAngle;        /* degrees (spot); negative: kPolymorphicLightShapingUseMinFalloff */
    uint32_t _pad;
} RtxptLightDesc;               /* 60 bytes */

typedef struct RtxptSceneDesc {
    const RtxptInstanceData*    instances;      uint32_t instanceCount;
    const RtxptGeometryData*    geometries;     uint32_t geometryCount;
    const RtxptSubInstanceData* subInstances;   uint32_t subInstanceCount;
    const RtxptMaterialData*    materials;      uint32_t materialCount;
    const RtxptBufferDesc*      buffers;        uint32_t bufferCount;
    const RtxptTextureDesc*     textures;       uint32_t textureCount;
    RtxptEnvCubeDesc            envCube;
    const RtxptLightDesc*       lights;         uint32_t lightCount;      /* analytic lights; may be NULL / 0 */
} RtxptSceneDesc;

/* ------------------------------------------------------------------------------------------------------------------
 * Per-frame constants: the slice of SampleConstants (Rtxpt/Shaders/SampleConstantBuffer.h:46-60) the reference-mode
 * dispatch reads.
 * ---------------------------------------------------------------------------------------------------------------- */

/* Rtxpt/Shaders/PathTracer/PathTracerShared.h:24-44 (112 bytes) */
typedef struct RtxptCameraData {
    float    PosW[3];       float NearZ;
    float    DirectionW[3]; float PixelConeSpreadAngle;
    float    CameraU[3];    float FarZ;
    float    CameraV[3];    float FocalDistance;
    float    CameraW[3];    float AspectRatio;
    uint32_t ViewportSize[2];
    float    ApertureRadius;
    float    _padding0;
    float    Jitter[2];
    float    _padding1, _padding2;
} RtxptCameraData;

/* Rtxpt/Shaders/PathTracer/Lighting/EnvMap.hlsli:24-31 ; transforms row-major float3x4 */
typedef struct RtxptEnvMapSceneParams {
    float Transform[12];
    float InvTransform[12];
    float ColorMultiplier[3];
    float Enabled;
} RtxptEnvMapSceneParams;

/* Subset of PathTracerConstants (Rtxpt/Shaders/PathTracer/PathTracerShared.h:47-104) that reference mode reads,
 * filled the way Sample::UpdatePathTracerConstants does (Rtxpt/Sample.cpp:1464-1556). */
typedef struct RtxptPathTracerConstants {
    uint32_t imageWidth, imageHeight;
    uint32_t sampleBaseIndex;               /* m_sampleIndex * ActualSamplesPerPixel() (Sample.cpp:1507) */
    float    perPixelJitterAAScale;         /* 1 in reference mode with AccumulationAA (Sample.cpp:1501) */
    uint32_t bounceCount;
    uint32_t diffuseBounceCount;
    float    EnvironmentMapDiffuseSampleMIPLevel;
    float    texLODBias;
    float    fireflyFilterThreshold;        /* 0 disables (Sample.cpp:1518-1522) */
    uint32_t NEEEnabled;
    uint32_t NEEType;                       /* 0 uniform, 1 power, 2 NEE-AT (see NEEATFeedback) */
    uint32_t NEECandidateSamples;
    uint32_t NEEFullSamples;                /* light samples per path vertex, each with its own shadow ray (SampleUI "Full samples", 1 by default); values above 63 act as 63, 0
                                             * takes none.  N > 1: a path_trace launch batches max(1, maxSubSamplesPerLaunch / N) sub-samples, and the first trace allocates
                                             * about 56 B x N per path of such a launch (RTXPT_ERR_OUT_OF_MEMORY if that fails; the context keeps working with N = 1).
                                             * N > 1 with NEEType 2 and NEEATFeedback is refused (RTXPT_ERR_UNSUPPORTED): a visible sample's feedback draw would decide the
                                             * next sample's candidates. */
    uint32_t enableRussianRoulette;         /* PT_ENABLE_RUSSIAN_ROULETTE macro, Sample.cpp:988-1042 */
    uint32_t enableLDSamplerForBSDF;        /* RTXPT_ENABLE_LOW_DISCREPANCY_SAMPLER_FOR_BSDF */
    uint32_t nestedDielectricsQuality;      /* RTXPT_NESTED_DIELECTRICS_QUALITY: 0 off, 1 fast */
    RtxptCameraData camera;
    RtxptEnvMapSceneParams envMap;
    float    distantVsLocalImportance;      /* NEEAT_Distant_vs_Local_Importance (SampleUI.h:160), scaled by 0.0002 inside like LightsBaker.cpp:1029 */
    uint32_t NEEATFeedback;                 /* with NEEType 2: 0 = power-based global table only (what LightsBaker gives a first frame); 1 = temporal feedback: per-pixel light reservoirs filled by
                                             * NEE, usage-weighted global table and per-tile local samplers, advanced once per frame by rtxpt_b200_neeat_update_begin / _end (SURVEY §8f row 1) */
    uint32_t NEEATImportanceBoost;          /* with NEEATFeedback: LightsBaker's importance boosters (LightsBaker.h:245-249, both on in RTXPT's UI): bit 0 lights in / near the view frustum (needs
                                             * rtxpt_b200_set_view), bit 1 lights that got brighter since the last frame; 0 = neither */
    uint32_t useApproximateMIS;             /* the resolved RTXPT_USE_APPROXIMATE_MIS macro (Sample.cpp:1015): 0 = full light-vs-BSDF MIS, 1 = approximate MIS, in which the light's
                                             * selection x solid-angle pdf is replaced by the constant 3 on both sides and the BSDF side reads no light record (LightSampler.hlsli:271-280).
                                             * RTXPT resolves it as SampleUI::ActualUseApproximateMIS() = RealtimeMode ? NEEMISType != 0 : NEEMISType == 2 (SampleUI.h:135), and its
                                             * default NEEMISType 1 makes realtime mode approximate: pt.useApproximateMIS = m_ui.ActualUseApproximateMIS().  Values above 1 are refused
                                             * (RTXPT_ERR_INVALID_ARGUMENT).  rtxpt_b200_default_constants gives 0. */
} RtxptPathTracerConstants;

/* ------------------------------------------------------------------------------------------------------------------
 * Context
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct RtxptConfig {
    int32_t  deviceOrdinal;             /* CUDA device; -1 = current */
    uint32_t maxWidth, maxHeight;       /* render-target allocation (Rtxpt/SampleCommon/RenderTargets.cpp:159-175) */
    uint32_t maxSubSamplesPerLaunch;    /* how many sub-samples one path_trace call may batch into a single wavefront */
    uint32_t tileRank, tileWorld;       /* screen-tile partition for multi-GPU: this context renders tiles t with t % world == rank; 0,1 = whole frame */
    uint32_t tileSize;                  /* pixels, power of two, default 64 */
    uint32_t flags;                     /* RTXPT_CFG_* */
} RtxptConfig;

#define RTXPT_CFG_COUNT_TRAVERSAL_STEPS  1u   /* instrumented traversal: per-launch node/triangle counters (SURVEY §8d) */
#define RTXPT_CFG_NO_MATERIAL_SORT       2u   /* disable the per-bounce sort by material class (A/B measurement only) */
#define RTXPT_CFG_EXPORT_GUIDES          8u   /* write the reference-mode guide buffers (depth, motion vectors, throughput) at every path vertex */
#define RTXPT_CFG_NO_OPACITY_MASKS     16u   /* do not bake per-triangle opacity masks for alpha-tested geometry (A/B measurement; results are identical either way) */
#define RTXPT_CFG_TIME_KERNELS           4u   /* CUDA events around every kernel: fills RtxptStats.msTraceClosest/msTraceShadow/msShade/msOther */
#define RTXPT_CFG_REBLUR_UNTILED        32u   /* ReBLUR's HitDistReconstruction reads its 5x5 taps from global memory instead of the shared-memory tile (A/B measurement; results are
                                                 identical either way).  The environment variable RTXPT_REBLUR_TILED=0 does the same for every context of the process */

typedef struct rtxpt_ctx rtxpt_ctx;

/* Replaces device/pipeline creation: Sample::Init + CreateRTPipelines (Rtxpt/Sample.cpp:136-397, Rtxpt/AdvancedSample.cpp:35-46). */
RTXPT_API int rtxpt_b200_create(const RtxptConfig* config, rtxpt_ctx** outCtx);
RTXPT_API int rtxpt_b200_destroy(rtxpt_ctx* ctx);
RTXPT_API const char* rtxpt_b200_last_error(void);

/* Replaces scene upload + acceleration-structure build + material/light baking:
 *   Sample::CreateBlases/BuildTLAS (Rtxpt/Sample.cpp:1061-1240), MaterialsBaker::Update (Materials/MaterialsBaker.cpp:1019-1065),
 *   LightsBaker::UpdateBegin light list + weights + proxies (Lighting/LightsBaker.cpp:964-1327), EnvMapImportanceSamplingBaker. */
RTXPT_API int rtxpt_b200_upload_scene(rtxpt_ctx* ctx, const RtxptSceneDesc* scene);

/* Replaces writeBuffer(m_constantBuffer, &constants) (Rtxpt/Sample.cpp:2182).  Also re-bakes light weights when the
 * environment parameters changed. */
RTXPT_API int rtxpt_b200_set_constants(rtxpt_ctx* ctx, const RtxptPathTracerConstants* constants);

/* Stochastic texture filtering (RTXTF, External/Rtxtf; RTXPT_STOCHASTIC_TEXTURE_FILTERING_ENABLE = 1 in Rtxpt/Shaders/PathTracer/Config.h:95).  RTXPT passes STFFilterMode,
 * STFMagnificationMethod and STFGaussianSigma (Sample.cpp:1466-1495, :1549-1555).  With `enable` set, every material texture fetch of every path-tracer pass (reference, BUILD,
 * FILL) goes through STF_SamplerState::Texture2DSampleLevel at the ray-cone lambda: one stochastic integer mip and one stochastic texel of the filter at that mip, fetched at its
 * centre, with the vertex's uniform numbers drawn as PathTracerBridgeDonut.hlsli:637-652 draws them.  Alpha testing, opacity masks, the environment and the emissive bake do not
 * use the texture sampler in RTXPT either and are unaffected.  Off (the default) renders exactly as a context that never called this.
 *   filterType:          STF_FILTER_TYPE_POINT 0, LINEAR 1, CUBIC 2, GAUSSIAN 3 (STFDefinitions.h); anything else is RTXPT_ERR_INVALID_ARGUMENT
 *   magnificationMethod: STF_MAGNIFICATION_METHOD_NONE 0 only, RTXPT's default.  Methods 1-6 (2x2 quad / fine / fine temporal, 3x3 fine ALU / LUT, 4x4 fine) mix the texels of
 *                        neighbouring lanes through WaveReadLaneAt (_Tex2D2x2WaveImpl, _Tex2D3x3WaveImpl, _Tex2D4x4WaveImpl): their result depends on which paths share a wave,
 *                        which in a wavefront with class-sorted queues has no reproducible equivalent, so they are refused with RTXPT_ERR_UNSUPPORTED
 *   gaussianSigma:       the Gaussian's standard deviation in texels (0.3 in RTXPT's UI); must be finite and positive (RTXPT_ERR_INVALID_ARGUMENT), read for every filter type
 * A refused description leaves the context's setting as it was.  Applies from the next path_trace / path_trace_realtime. */
typedef struct RtxptStochasticTextureFiltering {
    uint32_t enable;
    uint32_t filterType;
    uint32_t magnificationMethod;
    float    gaussianSigma;
} RtxptStochasticTextureFiltering;
#define RTXPT_STF_FILTER_TYPE_POINT     0u
#define RTXPT_STF_FILTER_TYPE_LINEAR    1u
#define RTXPT_STF_FILTER_TYPE_CUBIC     2u
#define RTXPT_STF_FILTER_TYPE_GAUSSIAN  3u
RTXPT_API int rtxpt_b200_set_texture_filtering(rtxpt_ctx* ctx, const RtxptStochasticTextureFiltering* stf);

/* Debug views (RTXPT's m_ui.DebugView -> DebugConstants::debugViewType, DebugViewType in Rtxpt/Shaders/PathTracer/PathTracerDebug.hlsli:25-65; m_ui.DebugViewStablePlaneIndex ->
 * debugViewStablePlaneIndex, Sample.cpp:2160-2161).  A view other than DISABLED makes every path_trace / path_trace_realtime call first clear RTXPT_BUFFER_DEBUG_VIZ_F16 (RGBA16F,
 * width x height, allocated by the first such call; RTXPT's u_ShaderDebugVizTextureBuffer, which RTXPT clears when the accumulation restarts, Sample.cpp:1427) and then draw the view into it.  Drawing the
 * buffer over the output colour (RTXPT blends it over ProcessedOutputColor) is the host's job.  Nothing else a call computes changes with the view.
 *   FIRST_HIT_*:     surfaceDebugViz (PathTracerBridgeDonut.hlsli:457-510) at path vertex 1: in reference mode of the last sub-sample of the call (only the call's last launch
 *                    draws), in realtime mode of the BUILD pass.  Pixels whose camera ray misses keep the cleared value.  The shader ID is 0xFFFFFFFF for every surface (one
 *                    shader; RTXPT without RTXPT_SHADER_ID)
 *   DOMINANT_STABLE_PLANE_INDEX, STABLE_PLANE_VIRTUAL_RAY_LENGTH .. STABLE_PLANE_SPEC_RADIANCE, STABLE_RADIANCE: StablePlanesDebugViz (PathTracerDebug.hlsli:359-461) after the
 *                    FILL passes of path_trace_realtime; nothing is drawn in reference mode, which has no stable planes (Sample.cpp:2551).  The mouse crosshair is not drawn
 *   STABLE_PLANE_RELAXED_DISOCCLUSION .. STABLE_PLANE_DENOISER_VALIDATION: DENOISER_FINAL_MERGE's views (PostProcess.hlsl:633-681), drawn by rtxpt_b200_denoiser_final_merge
 *                    (and so by rtxpt_b200_denoise_realtime) for the plane it merges.  With the split, of the four pixels that land on one quadrant pixel the one of even
 *                    coordinates draws (RTXPT leaves it to the GPU).  NRD's validation layer is not part of this library: DENOISER_VALIDATION shows the combined denoised radiance
 *   stablePlaneIndex: 0..2 shows that plane, RTXPT_DEBUG_VIEW_STABLE_PLANE_SPLIT (-1 in RTXPT) the three planes in four half-resolution quadrants; with one active plane
 *                    plane 0 is shown, as Sample.cpp:2161 does.  Any other value is RTXPT_ERR_INVALID_ARGUMENT
 * Refused with RTXPT_ERR_UNSUPPORTED: DENOISER_GUIDE_* (the DLSS-RR guide buffers), VBUFFER_*, SECONDARY_SURFACE_*, RESTIR*, REGIR_* (RTXDI and the raster V-buffer, which this library does not have).  debugViewType >= RTXPT_DEBUG_VIEW_MAX_COUNT
 * is RTXPT_ERR_INVALID_ARGUMENT.  A refused description leaves the context's view as it was.  Applies from the next path_trace / path_trace_realtime. */
typedef struct RtxptDebugView {
    uint32_t debugViewType;                 /* RTXPT_DEBUG_VIEW_* */
    uint32_t stablePlaneIndex;
} RtxptDebugView;
#define RTXPT_DEBUG_VIEW_DISABLED                           0u
#define RTXPT_DEBUG_VIEW_DOMINANT_STABLE_PLANE_INDEX        1u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_VIRTUAL_RAY_LENGTH    2u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_MOTION_VECTORS        3u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_NORMALS               4u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_ROUGHNESS             5u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_SPEC_AVG              6u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_DIFF_BSDF_ESTIMATE    7u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_DIFF_RADIANCE         8u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_SPEC_BSDF_ESTIMATE    9u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_SPEC_RADIANCE         10u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_RELAXED_DISOCCLUSION  11u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_DIFF_RADIANCE_DENOISED 12u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_SPEC_RADIANCE_DENOISED 13u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_COMBINED_RADIANCE_DENOISED 14u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_VIEW_Z                15u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_THROUGHPUT            16u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_DENOISER_VALIDATION   17u
#define RTXPT_DEBUG_VIEW_STABLE_RADIANCE                    18u
#define RTXPT_DEBUG_VIEW_DENOISER_GUIDE_DEPTH               19u     /* .. DENOISER_GUIDE_PRIMARY_LAYER 28 */
#define RTXPT_DEBUG_VIEW_DENOISER_GUIDE_PRIMARY_LAYER       28u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_BARYCENTRICS             29u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_FACE_NORMAL              30u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_GEOMETRY_NORMAL          31u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_SHADING_NORMAL           32u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_SHADING_TANGENT          33u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_SHADING_BITANGENT        34u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_FRONT_FACING             35u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_THIN_SURFACE             36u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_DIFFUSE                  37u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_SPECULAR                 38u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_ROUGHNESS                39u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_METALLIC                 40u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_SHADER_ID                41u
#define RTXPT_DEBUG_VIEW_FIRST_HIT_MATERIAL_ID              42u
#define RTXPT_DEBUG_VIEW_VBUFFER_MOTION_VECTORS             43u     /* .. REGIR_INDIRECT_OUTPUT 53 */
#define RTXPT_DEBUG_VIEW_REGIR_INDIRECT_OUTPUT              53u
#define RTXPT_DEBUG_VIEW_MAX_COUNT                          54u
#define RTXPT_DEBUG_VIEW_STABLE_PLANE_SPLIT                 0xFFFFFFFFu
RTXPT_API int rtxpt_b200_set_debug_view(rtxpt_ctx* ctx, const RtxptDebugView* view);

/* Replaces the loop body of Sample::PathTrace (Rtxpt/Sample.cpp:2503-2517): setPushConstants({subSampleIndex}) +
 * dispatchRays(width,height), for subSampleCount consecutive sub-samples starting at firstSubSampleIndex, each followed
 * by the reference-mode accumulation (AccumulationPass::Render, Rtxpt/Sample.cpp:2770-2778) when accumulate != 0.
 * Asynchronous on `cudaStream` (a cudaStream_t, NULL = the context's own stream). */
RTXPT_API int rtxpt_b200_path_trace(rtxpt_ctx* ctx, uint32_t firstSubSampleIndex, uint32_t subSampleCount, int accumulate, void* cudaStream);

/* Resets the accumulation counter (Sample::PreUpdatePathTracing accumulation reset, Rtxpt/Sample.cpp:1416-1450). */
RTXPT_API int rtxpt_b200_reset_accumulation(rtxpt_ctx* ctx);

enum {
    RTXPT_BUFFER_OUTPUT_COLOR_F16   = 0,    /* u_OutputColor RGBA16F of the last sub-sample (ShaderResourceBindings.hlsli:24) */
    RTXPT_BUFFER_ACCUMULATED_F32    = 1,    /* AccumulatedRadiance RGBA32F (RenderTargets.cpp) */
    RTXPT_BUFFER_DEPTH_F32          = 2,    /* u_Depth R32F guide of the last sub-sample (PathTracerBridgeDonut.hlsli:1096-1153); 0 = nothing exported */
    RTXPT_BUFFER_MOTION_VECTORS_F16 = 3,    /* u_MotionVectors RGBA16F; zero in reference mode (PathTracer.hlsli:487,684) */
    RTXPT_BUFFER_THROUGHPUT_R11G11B10 = 4   /* u_Throughput R11G11B10_FLOAT: saturate(thp) at the last exported vertex, 0 on a miss */
};
/* Device→host copy of a render target; blocks until the work queued on the context has finished. */
RTXPT_API int rtxpt_b200_readback(rtxpt_ctx* ctx, int buffer, void* dst, size_t dstBytes);
/* Device pointer of a render target (for zero-copy interop: NCCL all-gather of radiance tiles, image diffs on device). */
RTXPT_API int rtxpt_b200_device_ptr(rtxpt_ctx* ctx, int buffer, void** outPtr, size_t* outBytes);
RTXPT_API int rtxpt_b200_synchronize(rtxpt_ctx* ctx);

/* One-call end-to-end frame through host memory: set_constants + path_trace(accumulate) + readback of the accumulated
 * image into `dstRGBA32F` (width*height*16 bytes). */
RTXPT_API int rtxpt_b200_render_frame(rtxpt_ctx* ctx, const RtxptPathTracerConstants* constants,
                                      uint32_t firstSubSampleIndex, uint32_t subSampleCount, void* dstRGBA32F, size_t dstBytes);

/* ------------------------------------------------------------------------------------------------------------------
 * Realtime mode: path-space decomposition into "stable planes" (SURVEY §8 row a17).  Replaces the three dispatches of
 * Sample::PathTrace in realtime mode (Rtxpt/Sample.cpp:2455-2521): RayGen_BUILD (PATH_TRACER_MODE_BUILD_STABLE_PLANES:
 * Whitted-style delta-only exploration, writes the planes, their guides and the stable radiance), subSampleCount x
 * RayGen_FILL (PATH_TRACER_MODE_FILL_STABLE_PLANES: noisy path tracing restarted from plane 0, radiance deposited per
 * plane with its specular share) and, with no denoiser, PostProcess NO_DENOISER_FINAL_MERGE
 * (Rtxpt/ProcessingPasses/PostProcess.hlsl:692-709) into u_OutputColor.
 * Data contract = the reference's own resources: StablePlane records (Rtxpt/Shaders/PathTracer/StablePlanes.hlsli:48-80) in
 * GenericTS addressing (8x8 Morton tiles, Rtxpt/Shaders/PathTracer/Utils/Utils.hlsli:320-362), the 4-layer R32_UINT header,
 * StableRadiance RGBA16F, SpecularHitT R32F (Rtxpt/SampleCommon/RenderTargets.cpp:62-141, :340-351).
 * ---------------------------------------------------------------------------------------------------------------- */
#define RTXPT_STABLE_PLANE_COUNT            3u              /* cStablePlaneCount */
#define RTXPT_STABLE_PLANE_MAX_VERTEX_INDEX 15u             /* cStablePlaneMaxVertexIndex */
#define RTXPT_STABLE_PLANE_INVALID_BRANCH   0xFFFFFFFFu     /* cStablePlaneInvalidBranchID: plane unused, its radiance is not valid */
typedef struct RtxptStablePlane {           /* 80 B, StablePlanes.hlsli:48-80 */
    float    RayOrigin[3];                  /* start of the last segment before the plane's surface */
    float    LastRayTCurrent;
    float    RayDir[3];
    float    SceneLength;                   /* total ray travel; +inf = the plane is a miss (sky) */
    uint32_t PackedThpAndMVs[3];            /* fp16 pairs: throughput << 16 | motion vector */
    uint32_t VertexIndexAndRoughness;       /* vertex index << 16 | fp16 roughness */
    uint32_t DenoiserPackedBSDFEstimate[3]; /* fp16 pairs: diffuse estimate << 16 | specular estimate */
    uint32_t PackedNormal;                  /* octahedral, 2 x 16 bit */
    uint32_t PackedNoisyRadianceAndSpecAvg[2]; /* fp16 x 4: radiance rgb, specular average */
    uint32_t FlagsAndVertexIndex;
    uint32_t PackedCounters;
} RtxptStablePlane;

typedef struct RtxptRealtimeConstants {     /* the realtime-mode fields of PathTracerConstants + the two views (Sample.cpp:1501-1540, :1464-1480) */
    uint32_t activeStablePlaneCount;        /* _activeStablePlaneCount, 1..3 */
    uint32_t maxStablePlaneVertexDepth;     /* min(UI value, 15, bounceCount) (Sample.cpp:1532) */
    uint32_t allowPrimarySurfaceReplacement;
    uint32_t subSampleCount;                /* ActualSamplesPerPixel(); invSubSampleCount = 1 / subSampleCount attenuates the noisy radiance */
    float    matWorldToClipNoOffset[16];    /* view.matWorldToClipNoOffset, row-major, row vector x matrix */
    float    prevMatWorldToClipNoOffset[16];/* previousView.matWorldToClipNoOffset */
    float    clipToWindowScale[2];          /* view.clipToWindowScale = (0.5 w, -0.5 h) */
    float    _pad[2];
} RtxptRealtimeConstants;

enum {
    RTXPT_BUFFER_STABLE_PLANES        = 5,  /* RtxptStablePlane[3 * planeStride], GenericTS addressing */
    RTXPT_BUFFER_STABLE_PLANES_HEADER = 6,  /* uint32 [4][height][width]: layers 0-2 branch IDs, layer 3 first-hit ray length (bits 2..31) | dominant plane index (bits 0..1) */
    RTXPT_BUFFER_STABLE_RADIANCE_F16  = 7,  /* RGBA16F: emission / sky seen along the delta tree, no noise */
    RTXPT_BUFFER_SPECULAR_HITT_F32    = 8   /* R32F: specular hit distance of the dominant plane (denoiser guide) */
};
RTXPT_API int rtxpt_b200_set_realtime(rtxpt_ctx* ctx, const RtxptRealtimeConstants* realtime);
/* BUILD + subSampleCount x FILL (+ the no-denoiser merge into RTXPT_BUFFER_OUTPUT_COLOR_F16 when mergeNoDenoiser != 0); asynchronous on `cudaStream`.
 * Depth / motion vectors / throughput guides are those of the dominant plane (PathTracerStablePlanes.hlsli:316-321, :404-408). */
RTXPT_API int rtxpt_b200_path_trace_realtime(rtxpt_ctx* ctx, int mergeNoDenoiser, void* cudaStream);
/* ---- Denoiser interface of realtime mode (SURVEY §8 row a18, RTXPT's side of it): what PostProcess.hlsl does around NRD for one stable plane
 * (Sample::Denoise, Rtxpt/Sample.cpp:2560-2618: for plane = active-1 .. 0 { prepare inputs; NRD; final merge }).
 *   prepare_inputs = DENOISER_PREPARE_INPUTS, ReBLUR variant (ProcessingPasses/PostProcess.hlsl:444-570): splits the plane's noisy radiance into its
 *     diffuse and specular parts, demodulates by the BSDF estimates, clamps, and writes NRD's inputs: viewZ R32F (FLT_MAX = sky), motion RGBA16F,
 *     normal+roughness R10G10B10A2 (octahedral normal, linear roughness: NRD_NORMAL_ENCODING 2 / NRD_ROUGHNESS_ENCODING 1, External/Nrd/CMakeLists.txt:29-30),
 *     diffuse / specular radiance (YCoCg) + normalised hit distance RGBA16F, disocclusion-threshold mix R8; with initWithStableRadiance it first sets
 *     the output colour to the stable radiance and clears the combined history-clamp relaxation.
 *   final_merge = DENOISER_FINAL_MERGE (PostProcess.hlsl:577-690): output colour += denoised diffuse * diffuse estimate + denoised specular * specular
 *     estimate for pixels that have a surface; the two denoised images are RGBA16F device buffers in NRD's output encoding (YCoCg + hit distance), e.g.
 *     OUT_DIFF_RADIANCE_HITDIST / OUT_SPEC_RADIANCE_HITDIST of an NRD instance - or the prepared inputs themselves for an identity denoiser. */
typedef struct RtxptDenoiserConstants {
    float matWorldToView[16];               /* view.matWorldToView, row-major, row vector x matrix */
    float hitDistanceParameters[4];         /* nrd::HitDistanceParameters A, B, C, D (NRDSettings.h:206-220; Sample.cpp:2174) */
    float preExposedGrayLuminance;          /* 1 without tone mapping (Sample.cpp:1516) */
    float denoiserRadianceClampK;           /* m_ui.DenoiserRadianceClampK (Sample.cpp:1525) */
    float stablePlanesSuppressPrimaryIndirectSpecularK;  /* 0 = off (Sample.cpp:1536) */
    float _pad;
} RtxptDenoiserConstants;
enum {
    RTXPT_BUFFER_DENOISER_VIEWSPACE_Z_F32        = 9,
    RTXPT_BUFFER_DENOISER_MOTION_VECTORS_F16     = 10,
    RTXPT_BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2 = 11,
    RTXPT_BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16 = 12,
    RTXPT_BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16 = 13,
    RTXPT_BUFFER_DENOISER_DISOCCLUSION_MIX_R8    = 14,
    RTXPT_BUFFER_COMBINED_HISTORY_CLAMP_RELAX_R8 = 15
};
/* DenoisingGuidesBaker::DenoiseSpecHitT (ProcessingPasses/DenoisingGuidesBaker.hlsl:53-115; Sample.cpp:2541-2543): 5x5 depth-aware spread of RTXPT_BUFFER_SPECULAR_HITT_F32, in place,
 * after rtxpt_b200_path_trace_realtime and before the denoiser reads the guide (rtxpt_b200_denoise_realtime runs it itself). */
RTXPT_API int rtxpt_b200_denoise_spec_hit_t(rtxpt_ctx* ctx, void* cudaStream);
RTXPT_API int rtxpt_b200_denoiser_prepare_inputs(rtxpt_ctx* ctx, uint32_t stablePlaneIndex, int initWithStableRadiance, const RtxptDenoiserConstants* constants, void* cudaStream);
RTXPT_API int rtxpt_b200_denoiser_final_merge(rtxpt_ctx* ctx, uint32_t stablePlaneIndex, const void* dDenoisedDiffRGBA16F, const void* dDenoisedSpecRGBA16F, void* cudaStream);    /* NULL, NULL = the images rtxpt_b200_reblur_denoise wrote */
/* ---- DLSS Ray Reconstruction's inputs (RTXPT's default realtime frame, RealtimeAA = 3): PostProcess DLSSRRDenoiserPrepareInputs, the DENOISER_DLSS_RR branch of
 * ProcessingPasses/PostProcess.hlsl:175-440 (Sample.cpp:2710-2757).  DLSS itself (Streamline / NGX) is the host's.  Run after rtxpt_b200_path_trace_realtime(ctx, 0, s) and
 * rtxpt_b200_denoise_spec_hit_t; per pixel it mixes the stable planes' guides by plane weights (throughput 0.2, equalisation 0.01, dominant plane +0.05), and writes
 *   RTXPT_BUFFER_OUTPUT_COLOR_F16      (stable radiance + noisy radiance of every plane that hit a surface, scaled so that its largest channel is at most brightnessClampK, 1)
 *   RTXPT_BUFFER_RR_*                  diffuse albedo (with the stable radiance's grey mix and a 0.05 floor), specular albedo, unit normal + roughness, and specular motion
 *                                      vectors: plane 0's reflection hit mirrored behind a planar reflector where specular hit distance > 1e-3 and mixed roughness < 0.25,
 *                                      RTXPT_BUFFER_MOTION_VECTORS_F16's xy elsewhere.
 * brightnessClampK: PathTracerConstants::DLSSRRBrightnessClampK, the value the shader compares against, as Sample.cpp:1526 computes it: the UI's DLSSRRBrightnessClampK
 * (SampleUI.h:218, default 4096) times PathTracerConstants::preExposedGrayLuminance - 4096 only without tone mapping (preExposedGrayLuminance 1, Sample.cpp:1516).  Finite and
 * positive: RTXPT turns a UI value <= 0 into 0, which blacks the colour out, and this call refuses it.  RTXPT_ERR_INVALID_ARGUMENT before the first realtime frame at the current image
 * size.  The four RR targets are allocated by the first call (and again after a resize); before it, readback / device_ptr refuse them. */
RTXPT_API int rtxpt_b200_dlss_rr_prepare_inputs(rtxpt_ctx* ctx, float brightnessClampK, void* cudaStream);
enum {
    RTXPT_BUFFER_RR_DIFFUSE_ALBEDO_R11G11B10      = 22,   /* RRDiffuseAlbedo (RenderTargets.cpp:185-197) */
    RTXPT_BUFFER_RR_SPECULAR_ALBEDO_R11G11B10     = 23,   /* RRSpecAlbedo */
    RTXPT_BUFFER_RR_NORMALS_ROUGHNESS_F16         = 24,   /* RRNormalsAndRoughness RGBA16F: world-space normal, linear roughness */
    RTXPT_BUFFER_RR_SPECULAR_MOTION_VECTORS_F16   = 25    /* RRSpecMotionVectors RG16F, pixels, current -> previous frame */
};

/* ---- Tone mapping / auto exposure (SURVEY §8f row 4; replaces ToneMappingPass::Render, Rtxpt/ToneMapper/ToneMappingPasses.cpp:230-360): log-luminance mean of the frame (auto exposure),
 * exposure, white balance / exposure-compensation colour transform, operator, clamp, sRGB encode into RTXPT_BUFFER_LDR_COLOR_RGBA8 (RTXPT's LdrColor, SRGBA8).  Field meanings and
 * defaults: ToneMappingParameters (ToneMappingPasses.h:36-60).  Unlike the reference, the luminance is that of the frame being mapped (no read-back latency, exact mean instead of a MIP chain). */
typedef struct RtxptToneMappingParams {
    uint32_t toneMapOperator;           /* 0 Linear, 1 Reinhard, 2 ReinhardModified, 3 HejiHableAlu, 4 HableUc2, 5 Aces */
    uint32_t clamped, autoExposure, enabled, whiteBalance;
    float exposureCompensation, exposureValueMin, exposureValueMax;   /* stops; min / max bound the auto-exposure factor */
    float whiteScale, whiteMaxLuminance, whitePoint;                   /* HableUc2 white; ReinhardModified white; colour temperature in K (1667..25000) */
    float filmSpeed, fNumber, shutter;                                 /* manual exposure (used when autoExposure == 0): ISO, f-number, reciprocal shutter time */
    float _pad[2];
} RtxptToneMappingParams;
enum { RTXPT_BUFFER_LDR_COLOR_RGBA8 = 19 };
/* sourceBuffer: RTXPT_BUFFER_OUTPUT_COLOR_F16 (a frame) or RTXPT_BUFFER_ACCUMULATED_F32 (the reference-mode accumulation) */
RTXPT_API int rtxpt_b200_tone_map(rtxpt_ctx* ctx, const RtxptToneMappingParams* params, int sourceBuffer, void* cudaStream);
RTXPT_API int rtxpt_b200_tone_map_average_luminance(rtxpt_ctx* ctx, float* outAvgLuminance);        /* of the last rtxpt_b200_tone_map; waits for it */
/* host helper: ToneMappingPass::GetPreExposedGray (what RtxptDenoiserConstants::preExposedGrayLuminance is the luminance of, Sample.cpp:1516) */
RTXPT_API int rtxpt_b200_tone_map_pre_exposed_gray(const RtxptToneMappingParams* params, float avgLuminance, float* outRgb);

/* ---- Rigid-instance animation (SURVEY §8f row 4; stands in for the per-frame BLAS / TLAS update behind Sample::UpdateAccelStructs and BuildTLAS, Rtxpt/Sample.cpp:1170-1240): new
 * row-major 3x4 matrices for every instance of the uploaded scene; on the stream, the leaf triangles are re-transformed (one thread each) and the 8-wide BVH is refitted bottom-up,
 * level by level, with the builder's own quantisation - unmoved geometry gives back the built nodes bit for bit, topology never changes (quality degrades with large deformation:
 * rtxpt_b200_rebuild_bvh then).  The instance table keeps the previous call's matrices as InstanceData.prevTransform: the BUILD pass's motion vectors are those of the moved surface (BridgeDonut:631,
 * PathTracerStablePlanes.hlsli:282-291); call it every frame, as Sample does its TLAS update, so that an instance that stopped reports no motion.  Emissive triangles are baked into the
 * light list at upload: instances that carry them stay put (or re-upload). */
RTXPT_API int rtxpt_b200_update_instance_transforms(rtxpt_ctx* ctx, const float* transforms3x4, uint32_t instanceCount, void* cudaStream);
/* Rebuild of the 8-wide BVH on the GPU over the leaf triangles as they are now (after refits and skin updates), replacing the context's tree: what a DXR caller gets from a build
 * without the update flag, where rtxpt_b200_update_instance_transforms is the update.  PLOC clustering over Morton-sorted triangles, the same 8-wide collapse, slot assignment and
 * quantisation as the host builder.  The triangle set, gids, flags and opacity-mask slots stay; only the tree and the leaf order change.  The result is a function of the triangles alone
 * (not of their current leaf order) and is the same in both libraries.  The work is enqueued on the stream, and the call waits for that stream after every clustering iteration
 * and every tree level (to read back a count of a few bytes) and once at the end: it returns with the new tree in place.  Scratch memory is owned by the context and only grows
 * (a few hundred bytes per triangle).  RTXPT_ERR_NO_SCENE before an upload; an empty scene is a no-op; RTXPT_ERR_UNSUPPORTED when the tree would be deeper than 32 levels (the
 * traversal stack); on any error the previous tree stays.  Work that reads the tree must be ordered with this call on the stream, as with the refit. */
RTXPT_API int rtxpt_b200_rebuild_bvh(rtxpt_ctx* ctx, void* cudaStream);
/* Skinned meshes (Donut's skinning pass, External/Donut/shaders/skinning_cs.hlsl, which RTXPT runs before its BLAS updates, Sample.cpp:1170-1198): register a geometry's bind pose once
 * (vertex order = the geometry's vertex buffer; normals / tangents snorm8 x 4 as in the vertex buffer, may be NULL; four uint16 joint indices and four float weights per vertex), then per
 * frame hand the joint matrices (row-major 4x4, row vector x matrix, as Donut's t_JointMatrices): the vertices are blended on the stream and the path tracer's per-triangle shade
 * records (object-space positions, normals, tangents) rewritten from them.  Follow with rtxpt_b200_update_instance_transforms to refit the BVH.  The corners the records held before the
 * update become the geometry's previous-position stream (Donut's GeometryData.prevPositionOffset, which a scene may also bring along at upload): the BUILD pass's motion vectors of
 * a skinned surface are prevTransform x previous position - transform x position, as in the reference. */
typedef struct RtxptSkinDesc {
    uint32_t instanceIndex, geometryIndexInInstance, numVertices, _pad;
    const float* positions; const uint32_t* normals; const uint32_t* tangents; const uint16_t* jointIndices; const float* jointWeights;
} RtxptSkinDesc;
RTXPT_API int rtxpt_b200_skin_register(rtxpt_ctx* ctx, const RtxptSkinDesc* desc, uint32_t* outSkinId);
RTXPT_API int rtxpt_b200_skin_update(rtxpt_ctx* ctx, uint32_t skinId, const float* jointMatrices4x4, uint32_t numJoints, void* cudaStream);
/* tests / debugging: what = 0 BVH nodes (80 B each), 1 leaf triangles (48 B), 2 per-triangle shade records (96 B, by global triangle id),
 * 3 previous-position records (36 B), 4 instance table (RtxptInstanceData), 5 BVH level starts (uint32, levelCount + 1),
 * 6 exact node boxes of the last refit (6 floats per node; empty before the first refit), 7 the environment cube's MIP chain (the layout rtxpt_b200_bake_env_map returns; empty
 * without a cube), 8 the 1024^2 radiance / importance MIP chain (RGBA32F, MIPs back to back), 9 the environment lookup map (1024^2 uint32 light indices; empty while the environment
 * is disabled).  dst == NULL returns the size in *outBytes; synchronises the context's stream. */
RTXPT_API int rtxpt_b200_debug_scene_readback(rtxpt_ctx* ctx, int what, void* dst, size_t dstBytes, size_t* outBytes);
/* host-only inspection of the builder: the compressed BVH over a triangle soup (nodes 80 B, leaf triangles 48 B with gid = soup index, level ranges); call with NULL outputs for sizes */
RTXPT_API int rtxpt_b200_debug_build_bvh(const float* triangleVertices, uint32_t triangleCount, void* outNodes, void* outTris, uint32_t* outLevelStart,
                                         uint32_t* outNodeCount, uint32_t* outTriCount, uint32_t* outLevelCount);

/* ---- Environment-map baking (SURVEY §8f row 3; replaces EnvMapBaker::Update's BaseLayerCS / MIPReduceCS passes, Rtxpt/Lighting/Distant/EnvMapBaker.cpp:425-600, .hlsl:64-356): an
 * equirectangular or cube source and up to 16 directional lights (Sample.cpp collects the scene's DirectionalLights for it) are baked on the GPU into the RGBA16F cube the path tracer
 * samples, with the MIP chain's solid-angle weights.  The result is returned in host memory in the layout RtxptEnvCubeDesc takes (MIP m: 6 faces of (cubeDim >> m)^2 RGBA32F texels,
 * faces +x -x +y -y +z -z, values fp16-representable), ready for rtxpt_b200_upload_scene.  Not built: the procedural sky and the BC6U compression of the baked cube. */
typedef struct RtxptEnvBakeLight { float colorIntensity[4]; float direction[3]; float angularSize; } RtxptEnvBakeLight;   /* colour, W/sr; incoming direction; radians */
typedef struct RtxptEnvBakeDesc {
    uint32_t cubeDim;                   /* power of two, 2..4096 (EnvMapBaker: 2048, 1024 with the procedural sky) */
    uint32_t sourceType;                /* 0 none, 1 equirectangular, 2 cube */
    uint32_t sourceWidth, sourceHeight; /* cube: face size in sourceWidth */
    const float* source;                /* host, RGBA32F; cube: 6 faces back to back */
    float scaleColor[3];                /* BakeSettings::EnvMapRadianceScale */
    uint32_t directionalLightCount;
    RtxptEnvBakeLight lights[16];
} RtxptEnvBakeDesc;
RTXPT_API uint32_t rtxpt_b200_env_bake_mip_count(uint32_t cubeDim);
RTXPT_API size_t   rtxpt_b200_env_bake_floats(uint32_t cubeDim);          /* all MIPs back to back */
RTXPT_API int      rtxpt_b200_bake_env_map(rtxpt_ctx* ctx, const RtxptEnvBakeDesc* desc, float* outAllMips, size_t outFloats);
/* Re-bakes the environment of a live context on the GPU (EnvMapBaker::Update when it reports contentsChanged: the sun moved, the environment map was switched): the bake goes
 * straight into the cube the path tracer samples, the 1024^2 radiance / importance map (EnvMapImportanceSamplingBaker) is rebuilt from it on the GPU, and the environment's
 * quad-tree lights, lookup map, weights and proxy table are re-baked on the host from that map.  Only the importance map (~22 MB) crosses to the host; nothing else of the scene is
 * touched (BVH, skins, instance table, emissive triangles stay as they are).  Validation is that of rtxpt_b200_bake_env_map, except that source == NULL with sourceType 1 or 2
 * re-bakes from the source the context kept from its last update (same type and size, else RTXPT_ERR_INVALID_ARGUMENT).  cubeDim may differ from the uploaded cube; a scene
 * uploaded without a cube gains one.  On failure the previous cube, importance map and light list stay.  Like rtxpt_b200_update_lights: waits for the context's work in flight,
 * returns with the new light list on the device when constants are set (otherwise rtxpt_b200_set_constants uploads it), and NEE-AT's next update_begin maps last frame's feedback
 * onto the new environment nodes.  The importance map of an update and of an upload are built by the same arithmetic on GPU and host, but the GPU's cos / sin round differently
 * from the C library's in a small share of taps, so the two maps differ in a small share of texels. */
RTXPT_API int      rtxpt_b200_update_env_map(rtxpt_ctx* ctx, const RtxptEnvBakeDesc* desc, void* cudaStream);
/* event times of the last rtxpt_b200_update_env_map in ms: bake, importance map, copy into the cube array, read-back + host light bake + upload */
RTXPT_API int      rtxpt_b200_last_env_update_ms(rtxpt_ctx* ctx, float* outMs4);

/* ---- NEE-AT temporal feedback (SURVEY §8f row 1; replaces the feedback half of Rtxpt/Lighting/LightsBaker: UpdateBegin's ProcessFeedbackHistoryPreFilter / P0 + usage-weighted
 * ComputeProxyCounts, UpdateEnd's P1a / P1b / P2 / P3 / ClearFeedbackHistory, LightsBaker.cpp:1203-1225, :1331-1418).  Active with NEEType == 2 && NEEATFeedback != 0: NEE then draws
 * ComputeCandidateSampleLocalCount( 0.65, NEECandidateSamples ) of its candidates from the pixel's 8x8-tile sampler once a frame of feedback exists, mixes them with the global ones by
 * MIS, and records which light each pixel wanted.  Per frame: set_constants; neeat_update_begin; neeat_update_end (rtxpt_b200_path_trace_realtime calls it itself after its BUILD
 * pass; reference mode: call it before rtxpt_b200_path_trace - it reprojects with the guides the previous frame exported, so the context needs RTXPT_CFG_EXPORT_GUIDES); then
 * trace.  Sub-samples of a reference-mode call run one per wavefront while feedback is active (a pixel's reservoir is updated by one path at a time, as in the reference).
 * Single GPU: the tile partition does not carry the reservoirs. */
RTXPT_API int rtxpt_b200_neeat_update_begin(rtxpt_ctx* ctx, void* cudaStream);
RTXPT_API int rtxpt_b200_neeat_update_end(rtxpt_ctx* ctx, void* cudaStream);
/* Dynamic analytic lights: replaces the scene's light array (RtxptSceneDesc.lights) - lights that move, change colour / intensity / cone, are added at the end or dropped from the
 * end keep their identity by position in the array; the library re-bakes its light list (environment nodes, analytic lights, emissive triangles) as LightsBaker::UpdateBegin does
 * every frame.  With NEE-AT feedback active the reservoirs and tile samplers of the last frame follow the lights through the past -> current index tables of the reference
 * (LightsBaker.hlsl u_historyRemapPastToCurrent / CurrentToPast: environment nodes through the importance-map lookups, triangles by block offset); a removed light's feedback is
 * dropped.  Call before rtxpt_b200_neeat_update_begin of the frame.  Emissive geometry stays that of the upload; the environment changes through rtxpt_b200_update_env_map. */
RTXPT_API int rtxpt_b200_update_lights(rtxpt_ctx* ctx, const RtxptLightDesc* lights, uint32_t lightCount);
RTXPT_API int rtxpt_b200_neeat_reset(rtxpt_ctx* ctx);                 /* LightsBaker::BakeSettings::ResetFeedback: drop all feedback state */
/* tests / debugging: what = 0,1 feedback weight / candidate; 2,3 processed; 4,5 half-resolution blend; 6 tile lists; 7 proxy counters; 8 control words; 11 proxy table */
RTXPT_API int rtxpt_b200_neeat_readback(rtxpt_ctx* ctx, int what, void* dst, size_t dstBytes, size_t* outBytes);
RTXPT_API int rtxpt_b200_neeat_debug_set_feedback(rtxpt_ctx* ctx, const float* weight, const uint32_t* candidate);

/* ---- ReBLUR: NRD's REBLUR_DIFFUSE_SPECULAR denoiser (SURVEY §8 row a18; External/Nrd, NRD 4.15.2) for one stable plane, in RTXPT's configuration
 * (Rtxpt/NRD/NrdConfig.cpp:49-61 settings, NrdIntegration.cpp:375-408 common settings).  Replaces NrdIntegration::RunDenoiserPasses (NrdIntegration.cpp:360-520) for the
 * ReBLUR method: reads RTXPT_BUFFER_DENOISER_* as rtxpt_b200_denoiser_prepare_inputs wrote them, keeps one history per plane inside the context (RTXPT: one NRD instance per
 * plane), writes RTXPT_BUFFER_DENOISED_{DIFF,SPEC}_RADIANCE_HITDIST_F16 (NRD's OUT_DIFF/SPEC_RADIANCE_HITDIST), which rtxpt_b200_denoiser_final_merge( .., NULL, NULL ) consumes. */
typedef struct RtxptReblurFrame {
    float matWorldToView[16], matViewToClip[16];           /* this frame, un-jittered; row-major, row vector x matrix; left-handed view space, +z forward (nrd::CommonSettings::worldToViewMatrix / viewToClipMatrix) */
    float prevMatWorldToView[16], prevMatViewToClip[16];   /* previous frame (…MatrixPrev); equal to the current ones on the first frame */
    uint32_t frameIndex;                                    /* CommonSettings::frameIndex */
    uint32_t resetHistory;                                  /* AccumulationMode::CLEAR_AND_RESTART */
    uint32_t ignoreMotionVectors;                           /* 1: treat IN_MV as zero (static camera tests) */
    float frameTimeMs;                                      /* 0 = 1/60 s */
    float disocclusionThreshold, disocclusionThresholdAlternate;   /* 0 = RTXPT's UI defaults 0.03 / 0.2 (SampleUI.h:294-296) */
    float _pad[2];
} RtxptReblurFrame;
enum {
    RTXPT_BUFFER_DENOISED_DIFF_RADIANCE_HITDIST_F16 = 16,
    RTXPT_BUFFER_DENOISED_SPEC_RADIANCE_HITDIST_F16 = 17,
    RTXPT_BUFFER_REBLUR_ACCUMULATED_FRAMES_RG8      = 18   /* NRD's DATA1 after TemporalAccumulation: accumulated frames / 63 (diffuse, specular) */
};
RTXPT_API int rtxpt_b200_reblur_denoise(rtxpt_ctx* ctx, uint32_t stablePlaneIndex, const RtxptReblurFrame* frame, void* cudaStream);
/* ReBLUR settings: the nrd::ReblurSettings fields RTXPT's denoiser panel sets (Denoiser -> Advanced Settings, Rtxpt/SampleUI.cpp:1360-1410; m_ui.ReblurSettings, which Sample.cpp:2606-2610
 * hands to NrdIntegration::RunDenoiserPasses every frame) and m_ui.NRDUseAlternateDisocclusionThresholdMix (CommonSettings::isDisocclusionThresholdMixAvailable).
 * rtxpt_b200_default_reblur_settings gives NRD's defaults with RTXPT's overrides (NrdConfig.cpp:49-61): what a context uses until rtxpt_b200_set_reblur_settings is called.
 * rtxpt_b200_set_reblur_settings applies from the next reblur_denoise / denoise_realtime, to every plane's instance; as in NRD, a change keeps the history.  Refused with
 * RTXPT_ERR_INVALID_ARGUMENT, keeping the previous settings: a non-finite value, a negative radius, lobeAngleFraction / roughnessFraction / responsiveAccumulationRoughnessThreshold /
 * planeDistanceSensitivity outside [0, 1], a frame count above 63 (REBLUR_MAX_HISTORY_FRAME_NUM), a reconstruction mode above 2, a flag above 1.
 * hitDistanceParameters decode the normalised hit distances of the inputs.  As in RTXPT, which feeds one struct to both, the caller passes the same four values here and in
 * RtxptDenoiserConstants::hitDistanceParameters (which normalise them in rtxpt_b200_denoiser_prepare_inputs); the library does not check that they agree.
 * The passes follow NRD's dispatch graph (Reblur.cpp:117-160): hitDistanceReconstructionMode OFF skips HitDistReconstruction; both pre-pass radii 0 skip the PrePass. */
typedef struct RtxptReblurSettings {
    float hitDistanceParameters[4];                 /* HitDistanceParameters A, B, C, D (3, 0.1, 20, -25) */
    float antilagLuminanceSigmaScale;               /* antilagSettings.luminanceSigmaScale (4) */
    float antilagLuminanceSensitivity;              /* antilagSettings.luminanceSensitivity (3) */
    uint32_t maxAccumulatedFrameNum;                /* 50 (RTXPT) */
    uint32_t maxFastAccumulatedFrameNum;            /* 6 */
    uint32_t historyFixFrameNum;                    /* 3 */
    float diffusePrepassBlurRadius;                 /* pixels, 15 (RTXPT) */
    float specularPrepassBlurRadius;                /* pixels, 40 (RTXPT) */
    float minBlurRadius, maxBlurRadius;             /* pixels, 1 / 30 */
    float lobeAngleFraction, roughnessFraction;     /* 0.15 / 0.15 */
    float responsiveAccumulationRoughnessThreshold; /* 0 */
    float planeDistanceSensitivity;                 /* 0.02 */
    uint32_t hitDistanceReconstructionMode;         /* RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_* (AREA_5X5, RTXPT) */
    uint32_t enableAntiFirefly;                     /* 1 (RTXPT) */
    uint32_t useAlternateDisocclusionThresholdMix;  /* 1 (SampleUI.h:295): blend towards disocclusionThresholdAlternate by RTXPT_BUFFER_DENOISER_DISOCCLUSION_MIX_R8 */
} RtxptReblurSettings;
#define RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_OFF        0u
#define RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_3X3   1u
#define RTXPT_REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5   2u
RTXPT_API int rtxpt_b200_default_reblur_settings(RtxptReblurSettings* out);
RTXPT_API int rtxpt_b200_set_reblur_settings(rtxpt_ctx* ctx, const RtxptReblurSettings* settings);
/* Sample::Denoise for the ReBLUR method (Rtxpt/Sample.cpp:2560-2618): for plane = active-1 .. 0 { prepare_inputs (first: init with stable radiance); reblur_denoise; final_merge } */
RTXPT_API int rtxpt_b200_denoise_realtime(rtxpt_ctx* ctx, const RtxptDenoiserConstants* constants, const RtxptReblurFrame* frame, void* cudaStream);
/* device time (CUDA events on the call's stream) of the last rtxpt_b200_denoise_realtime; waits for it to finish */
RTXPT_API int rtxpt_b200_last_denoise_ms(rtxpt_ctx* ctx, float* outMs);

/* GenericTS addressing of the plane buffer (host helpers; Utils.hlsli:320-362) */
RTXPT_API uint32_t rtxpt_b200_generic_ts_line_stride(uint32_t width, uint32_t height);
RTXPT_API uint32_t rtxpt_b200_generic_ts_plane_stride(uint32_t width, uint32_t height);
RTXPT_API uint32_t rtxpt_b200_generic_ts_address(uint32_t x, uint32_t y, uint32_t plane, uint32_t lineStride, uint32_t planeStride);

typedef struct RtxptStats {
    uint64_t scatterRays;           /* closest-hit queries of the last path_trace call */
    uint64_t shadowRays;            /* any-hit (visibility) queries: one per valid light sample */
    uint64_t paths;
    uint64_t kernelLaunches;        /* kernels launched by the last path_trace call */
    uint64_t traversalNodeVisits;   /* closest-hit queries; only with RTXPT_CFG_COUNT_TRAVERSAL_STEPS */
    uint64_t traversalTriTests;
    uint64_t shadowNodeVisits;      /* any-hit queries */
    uint64_t shadowTriTests;
    uint64_t raysPerBounce[16];     /* scatter rays per wavefront iteration */
    float    msTotal;               /* CUDA-event time of the last path_trace call */
    float    msTraceClosest, msTraceShadow, msShade, msOther;     /* msOther: camera rays, commit and, with NEEFullSamples > 1, the NEE resolve */
    uint32_t bvhNodeCount, bvhTriangleCount;
    float    bvhBuildSeconds;
    uint32_t lightCount, lightProxyCount;
    uint32_t accumulatedSamples;
} RtxptStats;
RTXPT_API int rtxpt_b200_get_stats(rtxpt_ctx* ctx, RtxptStats* out);

/* Opacity masks: this implementation's equivalent of the reference's Opacity Micro-Maps (Rtxpt/OpacityMicroMap/: OC1_4_State OMMs baked per alpha-tested mesh and attached to
 * the BLAS, Rtxpt/SampleCommon/AccelerationStructureUtil.h:60-84).  upload_scene bakes 64 two-bit states (transparent / opaque / unknown) per alpha-tested triangle from mip 0 of
 * its alpha texture; the traversal kernels resolve candidates on known micro-triangles without the texture fetch of AlphaTestImpl (PathTracerBridgeDonut.hlsli:929-971).  A state is
 * "known" only where every possible bilinear tap agrees, so hits are bit-identical with RTXPT_CFG_NO_OPACITY_MASKS. */
typedef struct RtxptOpacityMaskStats {
    uint32_t triangles;                 /* alpha-tested triangles that carry a mask */
    uint32_t microTrianglesPerTriangle; /* 64 */
    uint64_t transparent, opaque, unknown;   /* micro-triangle states over the scene */
    float    bakeSeconds;
} RtxptOpacityMaskStats;
RTXPT_API int rtxpt_b200_get_opacity_mask_stats(rtxpt_ctx* ctx, RtxptOpacityMaskStats* out);
/* Host-only hooks of the baker (no CUDA device needed): the mask of one triangle with texture coordinates uv[3][2] over mip 0 (`format` RTXPT_FORMAT_*) of an alpha texture, and
 * the micro-triangle a barycentric hit (u, v) falls into (rtxpt_b200/csrc/opacity_masks.h). */
RTXPT_API int rtxpt_b200_host_bake_opacity_mask(const void* mip0, uint32_t width, uint32_t height, uint32_t format, uint32_t alphaCutoffByte, const float uv[6], uint32_t outMask[4]);
RTXPT_API uint32_t rtxpt_b200_host_opacity_micro_index(float u, float v);

/* ------------------------------------------------------------------------------------------------------------------
 * Multi-GPU tile exchange.  The reference is single-GPU (SURVEY §2.2); with RtxptConfig.tileWorld > 1 each context renders
 * the screen tiles t with t % tileWorld == tileRank.  pack_owned writes this context's accumulated pixels into a compact
 * device array of `paddedPixelsPerRank` float4 (the send buffer of an NCCL all-gather); unpack_all scatters the gathered
 * tileWorld * paddedPixelsPerRank float4 back into this context's full-frame accumulated image.
 * ---------------------------------------------------------------------------------------------------------------- */
RTXPT_API int rtxpt_b200_tile_layout(rtxpt_ctx* ctx, uint32_t* outOwnedPixels, uint32_t* outPaddedPixelsPerRank);
RTXPT_API int rtxpt_b200_pack_owned(rtxpt_ctx* ctx, void* dDst, void* cudaStream);
RTXPT_API int rtxpt_b200_unpack_all(rtxpt_ctx* ctx, const void* dSrcAll, void* cudaStream);
/* The realtime frame on several GPUs (SURVEY §8e, BASELINE configs[2]).  Every rank traces BUILD / FILL for the screen tiles it owns; what the frame needs of its neighbours is
 * exchanged as packed per-pixel images, one all-gather each, with the calls below (`buffers`: 1..8 RTXPT_BUFFER_* ids of plain per-pixel images of 1 / 4 / 8 / 16 bytes per pixel):
 *   1. rtxpt_b200_path_trace_realtime(ctx, 0, s)                                             own tiles
 *   2. exchange { DEPTH_F32, SPECULAR_HITT_F32, STABLE_PLANE_NEIGHBOUR_GUIDES }; rtxpt_b200_denoise_spec_hit_t      the 5x5 guide filter and the disocclusion relaxation of
 *      prepare_inputs (a pixel's four neighbours: branch ID + packed normal per plane, 24 B per pixel) read across tile borders
 *   3. per plane, last to first: rtxpt_b200_denoiser_prepare_inputs (own tiles); exchange the seven RTXPT_BUFFER_DENOISER_* / COMBINED_HISTORY_CLAMP_RELAX images;
 *      rtxpt_b200_reblur_denoise (whole frame, replicated: every rank keeps the same history); rtxpt_b200_denoiser_final_merge (own tiles)
 *   4. exchange { OUTPUT_COLOR_F16 }; rtxpt_b200_tone_map                                    auto exposure reads the whole frame
 * With DLSS-RR instead of ReBLUR, steps 3 and 4 become: rtxpt_b200_dlss_rr_prepare_inputs (own tiles); exchange { OUTPUT_COLOR_F16, RR_DIFFUSE_ALBEDO_R11G11B10,
 * RR_SPECULAR_ALBEDO_R11G11B10, RR_NORMALS_ROUGHNESS_F16, RR_SPECULAR_MOTION_VECTORS_F16 }: every rank then holds the whole RR set; DLSS-RR
 * also reads the whole frame's DEPTH_F32 (step 2's set) and MOTION_VECTORS_F16 (add it to step 2's set).
 * exchange = rtxpt_b200_exchange_pack into a send buffer of rtxpt_b200_exchange_bytes bytes, ncclAllGather (or torch.distributed.all_gather_into_tensor) into
 * tileWorld x that many bytes, rtxpt_b200_exchange_unpack.  With NEEATFeedback = 0 the assembled frame is bit-identical to the single-GPU frame (tests/test_gpu_multi.py); with
 * feedback every rank adapts on its own tiles (independent global tables, local samplers clamped at screen-tile borders: still unbiased, SURVEY §8e). */
enum { RTXPT_BUFFER_STABLE_PLANE_NEIGHBOUR_GUIDES = 20 };     /* exchange only: per plane { branch ID, StablePlane::PackedNormal } of every pixel */
enum { RTXPT_BUFFER_DEBUG_VIZ_F16 = 21 };     /* RGBA16F debug view (rtxpt_b200_set_debug_view); RTXPT_ERR_INVALID_ARGUMENT until a call with a view has allocated it */
RTXPT_API int rtxpt_b200_exchange_bytes(rtxpt_ctx* ctx, const int* buffers, uint32_t count, size_t* outBytesPerRank);
RTXPT_API int rtxpt_b200_exchange_pack(rtxpt_ctx* ctx, const int* buffers, uint32_t count, void* dDst, void* cudaStream);
RTXPT_API int rtxpt_b200_exchange_unpack(rtxpt_ctx* ctx, const int* buffers, uint32_t count, const void* dSrcAllRanks, void* cudaStream);

/* ------------------------------------------------------------------------------------------------------------------
 * Host-side glTF 2.0 loader (rtxpt_b200/csrc/gltf_loader.cpp): produces the RtxptSceneDesc tables from a .gltf / .glb
 * the way Donut's GltfImporter + Scene::CreateMeshBuffers and RTXPT's MaterialsBaker do on the reference's host side
 * (External/Donut/src/engine/GltfImporter.cpp:641-1430, Scene.cpp:821-1000, Rtxpt/Materials/MaterialsBaker.cpp:516-591,
 * :660-705, :960-1017).  Needs no CUDA device.  The returned object owns everything the desc points to.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct rtxpt_host_scene rtxpt_host_scene;
typedef struct RtxptGltfCamera {        /* perspective cameras found in the node graph, world space */
    float position[3], direction[3], up[3];
    float yfov, znear, zfar, aspectRatio;   /* radians; aspectRatio 0 = unspecified */
} RtxptGltfCamera;
/* What an RTXPT .scene.json carries besides geometry (Assets/<name>.scene.json; Donut Scene::LoadSceneGraph, External/Donut/src/engine/Scene.cpp:230-360, and the
 * leaf types of Rtxpt/SampleCommon/ExtendedScene.cpp:44-372): the environment light and the SampleSettings node.  All zero / empty for a plain glTF. */
typedef struct RtxptSceneFileInfo {
    char     environmentMapPath[260];   /* EnvironmentLight.path, relative to the media folder ('/' separators); "" = none */
    float    environmentRadianceScale[3];
    float    environmentRotation;       /* EnvironmentLight.rotation */
    uint32_t hasSampleSettings;
    uint32_t realtimeMode;              /* SampleSettings.realtimeMode (default true in the reference UI) */
    int32_t  maxBounces, maxDiffuseBounces;     /* -1 = not given */
    float    realtimeFireflyFilter, textureMIPBias;
    char     startingCamera[64];
    uint32_t modelCount, directionalLightCount; /* directional lights are folded into the environment map by the reference and are not in the light list */
} RtxptSceneFileInfo;
/* Loader option (process-wide, default off): keep BC1 / BC2 / BC3 / BC7 .dds textures block-compressed (RTXPT_FORMAT_BC*) instead of expanding them to RGBA8 on the host; BC4 / BC5
 * (one / two channels) are always expanded, their channel layout differs from what the material code reads. */
RTXPT_API void rtxpt_b200_loader_keep_block_compression(int enable);
RTXPT_API int rtxpt_b200_load_gltf(const char* path, rtxpt_host_scene** outScene);
/* Same, with RTXPT's material files applied on top of the glTF materials the way MaterialsBaker does (Rtxpt/Materials/MaterialsBaker.cpp:707-747, :868-917):
 * for a glTF material <name> of model file <model>.gltf the first existing of <sceneMaterialsDir>/<model>.<name>.material.json, <sceneMaterialsDir>/<name>.material.json,
 * <materialsDir>/<model>.<name>.material.json, <materialsDir>/<name>.material.json replaces it (either directory may be NULL). */
RTXPT_API int rtxpt_b200_load_gltf_ex(const char* path, const char* materialsDir, const char* sceneMaterialsDir, rtxpt_host_scene** outScene, uint32_t* outOverriddenMaterials);
/* RTXPT scene file: "models" (glTF paths relative to the media folder = the scene file's folder unless given), "graph" (named nodes with
 * translation / rotation (xyzw) | euler / scaling, "model" references - a model may be instanced several times -, children, and the leaf types PointLight,
 * SpotLight, DirectionalLight, EnvironmentLight, PerspectiveCamera[Ex], SampleSettings).  Material files are looked up under <media>/Materials and
 * <media>/Materials/<scene file stem> like MaterialsBaker does.  Animations, named "parent" links and game props are not read. */
RTXPT_API int rtxpt_b200_load_scene_json(const char* path, const char* mediaDir, rtxpt_host_scene** outScene);
RTXPT_API int rtxpt_b200_host_scene_info(const rtxpt_host_scene* scene, RtxptSceneFileInfo* outInfo);
RTXPT_API const char* rtxpt_b200_load_gltf_error(void);                 /* message of the last failed load on this thread */
RTXPT_API const RtxptSceneDesc* rtxpt_b200_host_scene_desc(const rtxpt_host_scene* scene);
RTXPT_API int rtxpt_b200_host_scene_cameras(const rtxpt_host_scene* scene, RtxptGltfCamera* outCameras, uint32_t* ioCount);
RTXPT_API uint32_t rtxpt_b200_host_scene_triangle_count(const rtxpt_host_scene* scene);
RTXPT_API void rtxpt_b200_free_host_scene(rtxpt_host_scene* scene);

/* RTXPT's own material files (Assets/Materials/<model>.<name>.material.json; PTMaterial::Read / FillData, Rtxpt/Materials/MaterialsBaker.cpp:160-245,
 * :516-591) -> PTMaterialData.  Texture slots come back unbound (indices 0xFFFFFFFF, Use*Texture flags clear) together with the paths the file names;
 * the caller (or rtxpt_b200_load_gltf_ex) binds what it can load.  In the reference these files override the glTF material of the same name. */
typedef struct RtxptMaterialJsonInfo {
    RtxptMaterialData data;
    uint32_t enableAlphaTesting, excludeFromNEE, skipRender, enableTransmission;
    uint32_t textureEnabled[5];         /* base, occlusion-roughness-metallic (or specular), normal, emissive, transmission: Enable*Texture && a path is given */
    uint32_t textureSRGB[5];
    char     texturePath[5][260];       /* relative to the media folder, '/' separators */
} RtxptMaterialJsonInfo;
RTXPT_API int rtxpt_b200_parse_material_json(const char* jsonText, RtxptMaterialJsonInfo* out);
RTXPT_API const char* rtxpt_b200_parse_material_json_error(void);

/* Host-side helpers every C/C++ caller needs (rtxpt_b200/csrc/host_helpers.cpp; no CUDA device required):
 * BridgeCamera (Rtxpt/Shaders/PathTracer/PathTracerShared.h:109-141; aspect ratio = width / height, jitter in pixels) and the
 * reference-mode defaults of Sample::UpdatePathTracerConstants with the SampleUI.h defaults (Rtxpt/Sample.cpp:1464-1556). */
RTXPT_API int rtxpt_b200_bridge_camera(uint32_t viewportWidth, uint32_t viewportHeight, const float camPos[3], const float camDir[3], const float camUp[3],
                                       float fovY, float nearZ, float farZ, float focalDistance, float apertureRadius, const float jitter[2], RtxptCameraData* out);
RTXPT_API int rtxpt_b200_default_constants(const RtxptCameraData* camera, int envMapPresent, RtxptPathTracerConstants* out);

/* The one matrix of SampleConstants.view (PlanarViewConstants) the reference-mode dispatch reads besides the camera block:
 * matWorldToClip, row-major, used as row-vector x matrix (Bridge::ExportSurface, PathTracerBridgeDonut.hlsli:1113-1115).
 * Only needed with RTXPT_CFG_EXPORT_GUIDES. */
/* host helper: the planar view's matrices of a BridgeCamera block (row-major, row vector x matrix; left-handed view space, +z forward; D3D clip space, z in [0, 1]) - what a host
 * without Donut's PlanarView needs for rtxpt_b200_set_view, RtxptRealtimeConstants, RtxptDenoiserConstants and RtxptReblurFrame.  Any output may be NULL. */
RTXPT_API int rtxpt_b200_camera_matrices(const RtxptCameraData* camera, float* outWorldToView16, float* outViewToClip16, float* outWorldToClip16);
typedef struct RtxptViewConstants { float matWorldToClip[16]; } RtxptViewConstants;
RTXPT_API int rtxpt_b200_set_view(rtxpt_ctx* ctx, const RtxptViewConstants* view);

/* ------------------------------------------------------------------------------------------------------------------
 * Inspection hooks used by the parity tests and the traversal micro-benchmark.  They run the same device code as
 * path_trace on caller-supplied work.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct RtxptRay  { float origin[3]; float tMin; float dir[3]; float tMax; } RtxptRay;   /* 32 bytes */
typedef struct RtxptHit  { float t; float u, v; uint32_t instanceIndex, geometryIndex, primitiveIndex; } RtxptHit; /* t<0: miss; (u,v) = weights of vertex 1 and 2 */

/* Closest-hit (anyHit=0) or first-hit (anyHit=1) queries for `count` host rays; alpha test included. */
RTXPT_API int rtxpt_b200_trace_rays(rtxpt_ctx* ctx, const RtxptRay* rays, uint32_t count, int anyHit, RtxptHit* outHits);
/* Same on device-resident rays, `repeat` launches back to back; returns the average kernel milliseconds (CUDA events). */
RTXPT_API int rtxpt_b200_trace_rays_device(rtxpt_ctx* ctx, const void* dRays, uint32_t count, int anyHit, void* dHits, uint32_t repeat, float* outMsPerLaunch);

/* Baked light list (PolymorphicLightInfo 32 B each), per-light proxy counters and the proxy index table. */
RTXPT_API int rtxpt_b200_get_lights(rtxpt_ctx* ctx, void* outLightInfos, uint32_t* ioLightCount,
                                    uint32_t* outProxyCounters, uint32_t* outProxyIndices, uint32_t* ioProxyCount);

/* PolymorphicLightInfoEx (16 B each: IesProfileIndex, PrimaryAxis, CosConeAngleAndSoftness, UniqueID) of the analytic lights, which
 * occupy light indices [5368, 5368 + count) between the environment quad-tree nodes and the emissive triangles. */
RTXPT_API int rtxpt_b200_get_lights_ex(rtxpt_ctx* ctx, void* outLightInfoEx, uint32_t* ioAnalyticLightCount);

/* Host-only: decodes one mip of a DDS file held in memory (BC1/2/3/4/5/7, RGBA8, BGRA8) into RGBA8 - what the loaders do with the DDS textures
 * RTXPT's assets and material files reference.  outRGBA may be NULL to query the size. */
RTXPT_API int rtxpt_b200_debug_decode_dds(const void* fileBytes, uint64_t fileSize, uint32_t mip, uint32_t* outWidth, uint32_t* outHeight, uint32_t* outMipCount, uint32_t* outSrgb,
                                          uint8_t* outRGBA, uint64_t outCapacity);
RTXPT_API const char* rtxpt_b200_debug_decode_dds_error(void);
/* Inspection hook: decodes a baseline / extended-sequential JPEG (8-bit, grey or YCbCr, any sampling factors, restart intervals) held in memory into RGBA8 - the decoder the
 * glTF loader uses for image/jpeg (the reference: stb_image through Donut's TextureCache).  Progressive, arithmetic-coded, 12-bit and CMYK files are refused with a message.
 * Call with outRGBA == NULL for the size.  Errors: rtxpt_b200_debug_decode_jpeg_error. */
RTXPT_API int rtxpt_b200_debug_decode_jpeg(const void* fileBytes, uint64_t fileSize, uint32_t* outWidth, uint32_t* outHeight, uint8_t* outRGBA, uint64_t outCapacity);
RTXPT_API const char* rtxpt_b200_debug_decode_jpeg_error(void);
/* HDR DDS files: the reference's environment maps (Assets/EnvironmentMaps/<name>_cube_bc6u.dds - BC6H_UF16 cubes read by Donut's DDSFile.cpp for EnvMapBaker,
 * Rtxpt/Lighting/Distant/EnvMapBaker.cpp:164-169).  BC6H UF16 / SF16, R16G16B16A16_FLOAT, R32G32B32A32_FLOAT; 2-D or cube.  Call with outRGBA32F == NULL for the sizes; then mip 0 of
 * every face comes back as RGBA32F, faces back to back in D3D order (+x -x +y -y +z -z): the `source` of RtxptEnvBakeDesc (sourceType 2).  Errors: rtxpt_b200_debug_decode_dds_error. */
RTXPT_API int rtxpt_b200_load_dds_hdr(const void* fileBytes, uint64_t fileSize, uint32_t* outWidth, uint32_t* outHeight, uint32_t* outFaces, uint32_t* outMipCount,
                                      float* outRGBA32F, uint64_t outCapacityFloats);

/* HDR image files by content: OpenEXR (single-part scan-line files; NONE / RLE / ZIPS / ZIP compression; HALF / FLOAT / UINT channels R G B A or Y), Radiance .hdr (RGBE, flat or
 * run-length coded) and the HDR DDS formats above.  These are the three kinds of file the reference lists as environment-map sources (Rtxpt/Sample.cpp:110-118, read through
 * External/Donut/src/engine/TextureCache.cpp:200-236); the EXR reader is also how an AccumulatedRadiance dump of an RTXPT run made elsewhere comes in for comparison (BASELINE.md,
 * scripts/compare_hdr_images.py).  Call with outRGBA32F == NULL for the sizes; rows come back top to bottom as RGBA32F (alpha 1 where the file has none; faces back to back for a
 * DDS cube, *outFaces = 6).  Errors: rtxpt_b200_load_hdr_image_error. */
RTXPT_API int rtxpt_b200_load_hdr_image(const void* fileBytes, uint64_t fileSize, uint32_t* outWidth, uint32_t* outHeight, uint32_t* outFaces, float* outRGBA32F, uint64_t outCapacityFloats);
RTXPT_API const char* rtxpt_b200_load_hdr_image_error(void);

/* Host-only: builds the compressed wide BVH over a triangle soup (9 floats per triangle) and reports its surface-area-heuristic statistics:
 * expected node visits / triangle tests of a random ray that hits the root box.  Used to judge builder changes without a GPU. */
typedef struct RtxptBvhStats { uint32_t nodeCount, triangleReferenceCount, leafCount, maxDepth; float expectedNodeVisits, expectedTriangleTests, buildSeconds, _pad; } RtxptBvhStats;
RTXPT_API int rtxpt_b200_debug_bvh_stats(const float* triangleVertices, uint32_t triangleCount, RtxptBvhStats* outStats);
/* The same statistics of the context's tree as it is now (after upload, refit or rebuild), over the root's current box; buildSeconds is the last build: the host build at upload or
 * the device rebuild (CUDA events).  Synchronises the context's stream and reads the nodes back. */
RTXPT_API int rtxpt_b200_get_bvh_stats(rtxpt_ctx* ctx, RtxptBvhStats* outStats);

/* StandardBSDF evaluated on the device for `count` records of 36 floats in / 16 floats out; see tests/test_bsdf_parity.py. */
RTXPT_API int rtxpt_b200_debug_bsdf(rtxpt_ctx* ctx, const float* in, uint32_t count, float* out);
/* Stateless sample generators evaluated on the device: out[i*8..] = 4 uniform + 4 low-discrepancy draws for
 * (pixelX,pixelY,vertexIndex,sampleIndex) tuples in `in` (4 u32 each). */
RTXPT_API int rtxpt_b200_debug_rng(rtxpt_ctx* ctx, const uint32_t* in, uint32_t count, uint32_t* out);
/* Leak checks: the number of CUDA resources (device arrays, streams, events, textures, pinned blocks) all contexts of the process hold right now.
 * Destroying a context returns it to what it was before the context was created. */
RTXPT_API int rtxpt_b200_debug_live_resources(uint64_t* out);

#ifdef __cplusplus
}
#endif
#endif /* RTXPT_B200_H_ */
