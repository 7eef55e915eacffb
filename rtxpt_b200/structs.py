"""ctypes mirrors of include/rtxpt_b200.h (the C ABI).  Layouts are byte-identical to the reference's GPU tables:
GeometryData / InstanceData (External/Donut/include/donut/shaders/bindless.h:28-70), SubInstanceData
(Rtxpt/Shaders/SubInstanceData.h:23-46), PTMaterialData (Rtxpt/Shaders/PathTracer/Materials/MaterialPT.h:45-80),
PathTracerCameraData / PathTracerConstants (Rtxpt/Shaders/PathTracer/PathTracerShared.h:24-104)."""
import ctypes as C
import math

u32, i32, f32, u64 = C.c_uint32, C.c_int32, C.c_float, C.c_uint64
MAX_MIPS = 16

FORMAT_RGBA8_UNORM, FORMAT_RGBA8_SRGB, FORMAT_RGBA32_FLOAT = 0, 1, 2
FORMAT_BC1_UNORM, FORMAT_BC1_SRGB, FORMAT_BC2_UNORM, FORMAT_BC2_SRGB, FORMAT_BC3_UNORM, FORMAT_BC3_SRGB, FORMAT_BC7_UNORM, FORMAT_BC7_SRGB = 3, 4, 5, 6, 7, 8, 9, 10
SUBINST_FLAG_ALPHA_TESTED = 1 << 16
SUBINST_FLAG_EXCLUDE_FROM_NEE = 1 << 17

MATFLAG_UseSpecularGlossModel = 0x1
MATFLAG_UseMetalRoughOrSpecularTexture = 0x4
MATFLAG_UseBaseOrDiffuseTexture = 0x8
MATFLAG_UseEmissiveTexture = 0x10
MATFLAG_UseNormalTexture = 0x20
MATFLAG_UseTransmissionTexture = 0x80
MATFLAG_MetalnessInRedChannel = 0x100
MATFLAG_ThinSurface = 0x200
MATFLAG_PSDExclude = 0x400
MATFLAG_EnableAsAnalyticLightProxy = 0x800
MATFLAG_IgnoreMeshTangentSpace = 1 << 12
MATFLAG_NestedPriorityShift = 28

CFG_COUNT_TRAVERSAL_STEPS = 1
CFG_NO_MATERIAL_SORT = 2
CFG_TIME_KERNELS = 4
CFG_EXPORT_GUIDES = 8
CFG_NO_OPACITY_MASKS = 16
CFG_REBLUR_UNTILED = 32

BUFFER_OUTPUT_COLOR_F16, BUFFER_ACCUMULATED_F32, BUFFER_DEPTH_F32, BUFFER_MOTION_VECTORS_F16, BUFFER_THROUGHPUT_R11G11B10 = 0, 1, 2, 3, 4
BUFFER_STABLE_PLANES, BUFFER_STABLE_PLANES_HEADER, BUFFER_STABLE_RADIANCE_F16, BUFFER_SPECULAR_HITT_F32 = 5, 6, 7, 8
STABLE_PLANE_COUNT, STABLE_PLANE_INVALID_BRANCH = 3, 0xFFFFFFFF
(BUFFER_DENOISER_VIEWSPACE_Z_F32, BUFFER_DENOISER_MOTION_VECTORS_F16, BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2, BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16,
 BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16, BUFFER_DENOISER_DISOCCLUSION_MIX_R8, BUFFER_COMBINED_HISTORY_CLAMP_RELAX_R8) = 9, 10, 11, 12, 13, 14, 15
BUFFER_DENOISED_DIFF_RADIANCE_HITDIST_F16, BUFFER_DENOISED_SPEC_RADIANCE_HITDIST_F16, BUFFER_REBLUR_ACCUMULATED_FRAMES_RG8 = 16, 17, 18
BUFFER_LDR_COLOR_RGBA8 = 19
BUFFER_STABLE_PLANE_NEIGHBOUR_GUIDES = 20        # exchange only (rtxpt_b200_exchange_*)
BUFFER_DEBUG_VIZ_F16 = 21                        # rtxpt_b200_set_debug_view
# DLSS-RR inputs (rtxpt_b200_dlss_rr_prepare_inputs)
BUFFER_RR_DIFFUSE_ALBEDO_R11G11B10, BUFFER_RR_SPECULAR_ALBEDO_R11G11B10, BUFFER_RR_NORMALS_ROUGHNESS_F16, BUFFER_RR_SPECULAR_MOTION_VECTORS_F16 = 22, 23, 24, 25
DLSS_RR_BRIGHTNESS_CLAMP_K = 4096.0              # PathTracerConstants::DLSSRRBrightnessClampK with RTXPT's UI default and tone mapping off; with it on, times preExposedGrayLuminance (Sample.cpp:1526)

class GeometryData(C.Structure):
    _fields_ = [("numIndices", u32), ("numVertices", u32), ("indexBufferIndex", i32), ("indexOffset", u32),
                ("vertexBufferIndex", i32), ("positionOffset", u32), ("prevPositionOffset", u32), ("texCoord1Offset", u32),
                ("texCoord2Offset", u32), ("normalOffset", u32), ("tangentOffset", u32), ("curveRadiusOffset", u32),
                ("materialIndex", u32), ("pad0", u32), ("pad1", u32), ("pad2", u32)]


class InstanceData(C.Structure):
    _fields_ = [("flags", u32), ("firstGeometryInstanceIndex", u32), ("firstGeometryIndex", u32), ("numGeometries", u32),
                ("transform", f32 * 12), ("prevTransform", f32 * 12)]


class SubInstanceData(C.Structure):
    _fields_ = [("FlagsAndAlphaInfo", u32), ("GlobalGeometryIndex_PTMaterialDataIndex", u32), ("EmissiveLightMappingOffset", u32),
                ("AnalyticProxyLightIndex", u32), ("IndexBufferIndex_VertexBufferIndex", u32), ("IndexOffset", u32),
                ("TexCoord1Offset", u32), ("padding0", u32)]


class MaterialData(C.Structure):
    _fields_ = [("BaseOrDiffuseColor", f32 * 3), ("Flags", u32), ("SpecularColor", f32 * 3), ("_padding0", i32),
                ("EmissiveColor", f32 * 3), ("ShadowNoLFadeout", f32), ("Opacity", f32), ("Roughness", f32), ("Metalness", f32),
                ("NormalTextureScale", f32), ("_padding1", f32), ("AlphaCutoff", f32), ("TransmissionFactor", f32),
                ("BaseOrDiffuseTextureIndex", u32), ("MetalRoughOrSpecularTextureIndex", u32), ("EmissiveTextureIndex", u32),
                ("NormalTextureIndex", u32), ("OcclusionTextureIndex", u32), ("TransmissionTextureIndex", u32), ("IoR", f32),
                ("ThicknessFactor", f32), ("DiffuseTransmissionFactor", f32), ("VolumeAttenuationColor", f32 * 3),
                ("VolumeAttenuationDistance", f32)]


class BufferDesc(C.Structure):
    _fields_ = [("data", C.c_void_p), ("sizeBytes", u64)]


class TextureDesc(C.Structure):
    _fields_ = [("width", u32), ("height", u32), ("mipLevels", u32), ("format", u32), ("mips", C.c_void_p * MAX_MIPS)]


class EnvCubeDesc(C.Structure):
    _fields_ = [("faceSize", u32), ("mipLevels", u32), ("faces", (C.c_void_p * MAX_MIPS) * 6)]


LIGHT_POINT, LIGHT_SPOT = 1, 2


class LightDesc(C.Structure):       # RtxptLightDesc, 60 bytes
    _fields_ = [("type", u32), ("position", f32 * 3), ("direction", f32 * 3), ("color", f32 * 3), ("intensity", f32), ("radius", f32),
                ("innerAngle", f32), ("outerAngle", f32), ("_pad", u32)]


class SceneDesc(C.Structure):
    _fields_ = [("instances", C.POINTER(InstanceData)), ("instanceCount", u32),
                ("geometries", C.POINTER(GeometryData)), ("geometryCount", u32),
                ("subInstances", C.POINTER(SubInstanceData)), ("subInstanceCount", u32),
                ("materials", C.POINTER(MaterialData)), ("materialCount", u32),
                ("buffers", C.POINTER(BufferDesc)), ("bufferCount", u32),
                ("textures", C.POINTER(TextureDesc)), ("textureCount", u32),
                ("envCube", EnvCubeDesc),
                ("lights", C.POINTER(LightDesc)), ("lightCount", u32)]


class MaterialJsonInfo(C.Structure):
    _fields_ = [("data", MaterialData), ("enableAlphaTesting", u32), ("excludeFromNEE", u32), ("skipRender", u32), ("enableTransmission", u32),
                ("textureEnabled", u32 * 5), ("textureSRGB", u32 * 5), ("texturePath", (C.c_char * 260) * 5)]


class BvhStats(C.Structure):
    _fields_ = [("nodeCount", u32), ("triangleReferenceCount", u32), ("leafCount", u32), ("maxDepth", u32), ("expectedNodeVisits", f32), ("expectedTriangleTests", f32),
                ("buildSeconds", f32), ("_pad", f32)]


class SceneFileInfo(C.Structure):
    _fields_ = [("environmentMapPath", C.c_char * 260), ("environmentRadianceScale", f32 * 3), ("environmentRotation", f32), ("hasSampleSettings", u32), ("realtimeMode", u32),
                ("maxBounces", C.c_int32), ("maxDiffuseBounces", C.c_int32), ("realtimeFireflyFilter", f32), ("textureMIPBias", f32), ("startingCamera", C.c_char * 64),
                ("modelCount", u32), ("directionalLightCount", u32)]


class GltfCamera(C.Structure):
    _fields_ = [("position", f32 * 3), ("direction", f32 * 3), ("up", f32 * 3), ("yfov", f32), ("znear", f32), ("zfar", f32), ("aspectRatio", f32)]


class ViewConstants(C.Structure):
    _fields_ = [("matWorldToClip", f32 * 16)]


class StablePlane(C.Structure):          # 80 B, StablePlanes.hlsli:48-80
    _fields_ = [("RayOrigin", f32 * 3), ("LastRayTCurrent", f32), ("RayDir", f32 * 3), ("SceneLength", f32), ("PackedThpAndMVs", u32 * 3), ("VertexIndexAndRoughness", u32),
                ("DenoiserPackedBSDFEstimate", u32 * 3), ("PackedNormal", u32), ("PackedNoisyRadianceAndSpecAvg", u32 * 2), ("FlagsAndVertexIndex", u32), ("PackedCounters", u32)]


STABLE_PLANE_DTYPE = [("RayOrigin", "f4", 3), ("LastRayTCurrent", "f4"), ("RayDir", "f4", 3), ("SceneLength", "f4"), ("PackedThpAndMVs", "u4", 3), ("VertexIndexAndRoughness", "u4"),
                      ("DenoiserPackedBSDFEstimate", "u4", 3), ("PackedNormal", "u4"), ("PackedNoisyRadianceAndSpecAvg", "u4", 2), ("FlagsAndVertexIndex", "u4"), ("PackedCounters", "u4")]


class DenoiserConstants(C.Structure):
    _fields_ = [("matWorldToView", f32 * 16), ("hitDistanceParameters", f32 * 4), ("preExposedGrayLuminance", f32), ("denoiserRadianceClampK", f32),
                ("stablePlanesSuppressPrimaryIndirectSpecularK", f32), ("_pad", f32)]


class SkinDesc(C.Structure):
    _fields_ = [("instanceIndex", u32), ("geometryIndexInInstance", u32), ("numVertices", u32), ("_pad", u32), ("positions", C.c_void_p), ("normals", C.c_void_p), ("tangents", C.c_void_p),
                ("jointIndices", C.c_void_p), ("jointWeights", C.c_void_p)]


class ToneMappingParams(C.Structure):
    _fields_ = [("toneMapOperator", u32), ("clamped", u32), ("autoExposure", u32), ("enabled", u32), ("whiteBalance", u32), ("exposureCompensation", f32), ("exposureValueMin", f32),
                ("exposureValueMax", f32), ("whiteScale", f32), ("whiteMaxLuminance", f32), ("whitePoint", f32), ("filmSpeed", f32), ("fNumber", f32), ("shutter", f32), ("_pad", f32 * 2)]


def make_tone_mapping_params(op=5, clamped=True, auto_exposure=False, enabled=True, white_balance=False, exposure_compensation=0.0, exposure_value_min=-16.0, exposure_value_max=16.0,
                             white_scale=11.2, white_max_luminance=1.0, white_point=6500.0, film_speed=100.0, f_number=1.0, shutter=1.0):
    """ToneMappingParameters with the defaults of ToneMappingPasses.h:36-60 (Aces, clamped, manual exposure that scales by 1)."""
    p = ToneMappingParams(); p.toneMapOperator = op; p.clamped = int(clamped); p.autoExposure = int(auto_exposure); p.enabled = int(enabled); p.whiteBalance = int(white_balance)
    p.exposureCompensation = exposure_compensation; p.exposureValueMin = exposure_value_min; p.exposureValueMax = exposure_value_max; p.whiteScale = white_scale
    p.whiteMaxLuminance = white_max_luminance; p.whitePoint = white_point; p.filmSpeed = film_speed; p.fNumber = f_number; p.shutter = shutter
    return p


class EnvBakeLight(C.Structure):
    _fields_ = [("colorIntensity", f32 * 4), ("direction", f32 * 3), ("angularSize", f32)]


class EnvBakeDesc(C.Structure):
    _fields_ = [("cubeDim", u32), ("sourceType", u32), ("sourceWidth", u32), ("sourceHeight", u32), ("source", C.c_void_p), ("scaleColor", f32 * 3), ("directionalLightCount", u32),
                ("lights", EnvBakeLight * 16)]


class ReblurFrame(C.Structure):
    _fields_ = [("matWorldToView", f32 * 16), ("matViewToClip", f32 * 16), ("prevMatWorldToView", f32 * 16), ("prevMatViewToClip", f32 * 16),
                ("frameIndex", u32), ("resetHistory", u32), ("ignoreMotionVectors", u32), ("frameTimeMs", f32),
                ("disocclusionThreshold", f32), ("disocclusionThresholdAlternate", f32), ("_pad", f32 * 2)]


class ReblurSettings(C.Structure):
    """RtxptReblurSettings (rtxpt_b200_set_reblur_settings): the nrd::ReblurSettings fields RTXPT's denoiser panel sets.  ReblurSettings.default() gives what a context uses
    until the setter is called (NRD's defaults with RTXPT's overrides)."""
    _fields_ = [("hitDistanceParameters", f32 * 4), ("antilagLuminanceSigmaScale", f32), ("antilagLuminanceSensitivity", f32),
                ("maxAccumulatedFrameNum", u32), ("maxFastAccumulatedFrameNum", u32), ("historyFixFrameNum", u32),
                ("diffusePrepassBlurRadius", f32), ("specularPrepassBlurRadius", f32), ("minBlurRadius", f32), ("maxBlurRadius", f32),
                ("lobeAngleFraction", f32), ("roughnessFraction", f32), ("responsiveAccumulationRoughnessThreshold", f32), ("planeDistanceSensitivity", f32),
                ("hitDistanceReconstructionMode", u32), ("enableAntiFirefly", u32), ("useAlternateDisocclusionThresholdMix", u32)]

    @classmethod
    def default(cls, **changes):
        """RTXPT's settings (rtxpt_b200_default_reblur_settings), with `changes` (field name = value) applied"""
        s = cls((f32 * 4)(3.0, 0.1, 20.0, -25.0), 4.0, 3.0, 50, 6, 3, 15.0, 40.0, 1.0, 30.0, 0.15, 0.15, 0.0, 0.02, REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5, 1, 1)
        for k, v in changes.items():
            if k == "hitDistanceParameters": s.hitDistanceParameters = (f32 * 4)(*v)
            else: setattr(s, k, v)
        return s


REBLUR_HIT_DISTANCE_RECONSTRUCTION_OFF, REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_3X3, REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5 = 0, 1, 2
REBLUR_MAX_HISTORY_FRAME_NUM = 63


def reblur_settings_status(s):
    """What rtxpt_b200_set_reblur_settings returns for `s`: 0, or RTXPT_ERR_INVALID_ARGUMENT (-1)"""
    # ctypes hands back the stored float32 values, so the comparisons below are the library's
    values = list(s.hitDistanceParameters) + [getattr(s, k) for k in ("antilagLuminanceSigmaScale", "antilagLuminanceSensitivity", "diffusePrepassBlurRadius",
              "specularPrepassBlurRadius", "minBlurRadius", "maxBlurRadius", "lobeAngleFraction", "roughnessFraction", "responsiveAccumulationRoughnessThreshold", "planeDistanceSensitivity")]
    if not all(math.isfinite(v) for v in values):
        return -1
    if min(s.diffusePrepassBlurRadius, s.specularPrepassBlurRadius, s.minBlurRadius, s.maxBlurRadius) < 0:
        return -1
    if not all(0 <= getattr(s, k) <= 1 for k in ("lobeAngleFraction", "roughnessFraction", "responsiveAccumulationRoughnessThreshold", "planeDistanceSensitivity")):
        return -1
    if max(s.maxAccumulatedFrameNum, s.maxFastAccumulatedFrameNum, s.historyFixFrameNum) > REBLUR_MAX_HISTORY_FRAME_NUM:
        return -1
    if s.hitDistanceReconstructionMode > REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_5X5 or s.enableAntiFirefly > 1 or s.useAlternateDisocclusionThresholdMix > 1:
        return -1
    return 0


class RealtimeConstants(C.Structure):
    _fields_ = [("activeStablePlaneCount", u32), ("maxStablePlaneVertexDepth", u32), ("allowPrimarySurfaceReplacement", u32), ("subSampleCount", u32),
                ("matWorldToClipNoOffset", f32 * 16), ("prevMatWorldToClipNoOffset", f32 * 16), ("clipToWindowScale", f32 * 2), ("_pad", f32 * 2)]


class CameraData(C.Structure):
    _fields_ = [("PosW", f32 * 3), ("NearZ", f32), ("DirectionW", f32 * 3), ("PixelConeSpreadAngle", f32),
                ("CameraU", f32 * 3), ("FarZ", f32), ("CameraV", f32 * 3), ("FocalDistance", f32),
                ("CameraW", f32 * 3), ("AspectRatio", f32), ("ViewportSize", u32 * 2), ("ApertureRadius", f32),
                ("_padding0", f32), ("Jitter", f32 * 2), ("_padding1", f32), ("_padding2", f32)]


class EnvMapSceneParams(C.Structure):
    _fields_ = [("Transform", f32 * 12), ("InvTransform", f32 * 12), ("ColorMultiplier", f32 * 3), ("Enabled", f32)]


class StochasticTextureFiltering(C.Structure):
    """RtxptStochasticTextureFiltering (rtxpt_b200_set_texture_filtering): filterType STF_FILTER_TYPE_* (0 point, 1 linear, 2 cubic, 3 Gaussian), magnificationMethod 0 only"""
    _fields_ = [("enable", u32), ("filterType", u32), ("magnificationMethod", u32), ("gaussianSigma", f32)]


STF_FILTER_POINT, STF_FILTER_LINEAR, STF_FILTER_CUBIC, STF_FILTER_GAUSSIAN = 0, 1, 2, 3


class DebugView(C.Structure):
    """RtxptDebugView (rtxpt_b200_set_debug_view): debugViewType is RTXPT's DebugViewType, stablePlaneIndex 0..2 or DEBUG_VIEW_STABLE_PLANE_SPLIT"""
    _fields_ = [("debugViewType", u32), ("stablePlaneIndex", u32)]


# DebugViewType (Rtxpt/Shaders/PathTracer/PathTracerDebug.hlsli:25-65), in order
DEBUG_VIEW_NAMES = (
    "Disabled", "DominantStablePlaneIndex",
    "StablePlane_VirtualRayLength", "StablePlane_MotionVectors", "StablePlane_Normals", "StablePlane_Roughness", "StablePlane_SpecAvg", "StablePlane_DiffBSDFEstimate",
    "StablePlane_DiffRadiance", "StablePlane_SpecBSDFEstimate", "StablePlane_SpecRadiance", "StablePlane_RelaxedDisocclusion", "StablePlane_DiffRadianceDenoised",
    "StablePlane_SpecRadianceDenoised", "StablePlane_CombinedRadianceDenoised", "StablePlane_ViewZ", "StablePlane_Throughput", "StablePlane_DenoiserValidation",
    "StableRadiance",
    "DenoiserGuide_Depth", "DenoiserGuide_Roughness", "DenoiserGuide_Albedo", "DenoiserGuide_SpecAlbedo", "DenoiserGuide_Normal", "DenoiserGuide_MotionVectors",
    "DenoiserGuide_SpecMotionVectors", "DenoiserGuide_SpecHitT", "DenoiserGuide_LayerWeights", "DenoiserGuide_PrimaryLayer",
    "FirstHit_Barycentrics", "FirstHit_FaceNormal", "FirstHit_GeometryNormal", "FirstHit_ShadingNormal", "FirstHit_ShadingTangent", "FirstHit_ShadingBitangent",
    "FirstHit_FrontFacing", "FirstHit_ThinSurface", "FirstHit_Diffuse", "FirstHit_Specular", "FirstHit_Roughness", "FirstHit_Metallic", "FirstHit_ShaderID", "FirstHit_MaterialID",
    "VBufferMotionVectors", "VBufferDepth",
    "SecondarySurfacePosition", "SecondarySurfaceRadiance", "ReSTIRGIOutput",
    "ReSTIRDIInitialOutput", "ReSTIRDITemporalOutput", "ReSTIRDISpatialOutput", "ReSTIRDIFinalOutput", "ReSTIRDIFinalContribution", "ReGIRIndirectOutput",
)
DEBUG_VIEW = {name: i for i, name in enumerate(DEBUG_VIEW_NAMES)}
DEBUG_VIEW_MAX_COUNT = len(DEBUG_VIEW_NAMES)
DEBUG_VIEW_STABLE_PLANE_SPLIT = 0xFFFFFFFF
DEBUG_VIEWS_FIRST_HIT = tuple(range(DEBUG_VIEW["FirstHit_Barycentrics"], DEBUG_VIEW["FirstHit_MaterialID"] + 1))
DEBUG_VIEWS_STABLE_PLANES = tuple(range(DEBUG_VIEW["DominantStablePlaneIndex"], DEBUG_VIEW["StablePlane_SpecRadiance"] + 1)) + (DEBUG_VIEW["StableRadiance"],)
DEBUG_VIEWS_DENOISER_MERGE = tuple(range(DEBUG_VIEW["StablePlane_RelaxedDisocclusion"], DEBUG_VIEW["StablePlane_DenoiserValidation"] + 1))


def debug_view_status(view, stable_plane_index=DEBUG_VIEW_STABLE_PLANE_SPLIT):
    """What rtxpt_b200_set_debug_view returns for a description: 0, or RTXPT_ERR_INVALID_ARGUMENT (-1) / RTXPT_ERR_UNSUPPORTED (-6)"""
    if not 0 <= view < DEBUG_VIEW_MAX_COUNT or not (0 <= stable_plane_index < 3 or stable_plane_index == DEBUG_VIEW_STABLE_PLANE_SPLIT):
        return -1
    return 0 if view == DEBUG_VIEW["Disabled"] or view in DEBUG_VIEWS_FIRST_HIT + DEBUG_VIEWS_STABLE_PLANES + DEBUG_VIEWS_DENOISER_MERGE else -6


class PathTracerConstants(C.Structure):
    _fields_ = [("imageWidth", u32), ("imageHeight", u32), ("sampleBaseIndex", u32), ("perPixelJitterAAScale", f32),
                ("bounceCount", u32), ("diffuseBounceCount", u32), ("EnvironmentMapDiffuseSampleMIPLevel", f32), ("texLODBias", f32),
                ("fireflyFilterThreshold", f32), ("NEEEnabled", u32), ("NEEType", u32), ("NEECandidateSamples", u32),
                ("NEEFullSamples", u32), ("enableRussianRoulette", u32), ("enableLDSamplerForBSDF", u32),
                ("nestedDielectricsQuality", u32), ("camera", CameraData), ("envMap", EnvMapSceneParams),
                ("distantVsLocalImportance", f32), ("NEEATFeedback", u32), ("NEEATImportanceBoost", u32), ("useApproximateMIS", u32)]


class Config(C.Structure):
    _fields_ = [("deviceOrdinal", i32), ("maxWidth", u32), ("maxHeight", u32), ("maxSubSamplesPerLaunch", u32),
                ("tileRank", u32), ("tileWorld", u32), ("tileSize", u32), ("flags", u32)]


class Stats(C.Structure):
    _fields_ = [("scatterRays", u64), ("shadowRays", u64), ("paths", u64), ("kernelLaunches", u64),
                ("traversalNodeVisits", u64), ("traversalTriTests", u64), ("shadowNodeVisits", u64), ("shadowTriTests", u64), ("raysPerBounce", u64 * 16),
                ("msTotal", f32), ("msTraceClosest", f32), ("msTraceShadow", f32), ("msShade", f32), ("msOther", f32),
                ("bvhNodeCount", u32), ("bvhTriangleCount", u32), ("bvhBuildSeconds", f32),
                ("lightCount", u32), ("lightProxyCount", u32), ("accumulatedSamples", u32)]


class OpacityMaskStats(C.Structure):
    _fields_ = [("triangles", u32), ("microTrianglesPerTriangle", u32), ("transparent", u64), ("opaque", u64), ("unknown", u64), ("bakeSeconds", f32)]


class Ray(C.Structure):
    _fields_ = [("origin", f32 * 3), ("tMin", f32), ("dir", f32 * 3), ("tMax", f32)]


class Hit(C.Structure):
    _fields_ = [("t", f32), ("u", f32), ("v", f32), ("instanceIndex", u32), ("geometryIndex", u32), ("primitiveIndex", u32)]


assert C.sizeof(GeometryData) == 64 and C.sizeof(InstanceData) == 112 and C.sizeof(SubInstanceData) == 32
assert C.sizeof(MaterialData) == 128 and C.sizeof(CameraData) == 112 and C.sizeof(Ray) == 32 and C.sizeof(Hit) == 24
