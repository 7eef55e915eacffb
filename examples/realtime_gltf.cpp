// realtime_gltf.cpp - the realtime side of the C ABI in one C++ host: load a glTF / .scene.json, then per frame what Sample::Render does around the realtime path tracer
// (Rtxpt/Sample.cpp:1412, :2438-2618, ToneMappingPasses.cpp:230-360): LightsBaker feedback update -> stable-plane BUILD + FILL -> guide filter + per-plane ReBLUR + final merge ->
// tone mapping; the last frame's SRGBA8 image is written as a PPM.  Static camera and scene (animation: rtxpt_b200_update_instance_transforms / rtxpt_b200_skin_update before the trace).
//   realtime_gltf scene.gltf out.ppm [width height frames bounces] [--approximate-mis]
// --approximate-mis: approximate light-vs-BSDF MIS, what RTXPT's realtime mode compiles by default (SampleUI NEEMISType 1: ActualUseApproximateMIS() is true in realtime mode)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "rtxpt_b200.h"

static int fail(const char* what, rtxpt_ctx* ctx) { fprintf(stderr, "%s: %s\n", what, ctx ? rtxpt_b200_last_error() : rtxpt_b200_load_gltf_error()); return 1; }
#define TRY(call) do { if ((call) != RTXPT_OK) return fail(#call, ctx); } while (0)

int main(int argc, char** argv)
{
    bool approximateMIS = false;
    for (int i = 1; i < argc; i++)
        if (!strcmp(argv[i], "--approximate-mis")) { approximateMIS = true; for (int j = i; j + 1 < argc; j++) argv[j] = argv[j + 1]; argc--; i--; }
    if (argc < 3) { fprintf(stderr, "usage: %s scene.gltf out.ppm [width height frames bounces] [--approximate-mis]\n", argv[0]); return 2; }
    const uint32_t width = argc > 3 ? uint32_t(atoi(argv[3])) : 512, height = argc > 4 ? uint32_t(atoi(argv[4])) : 512;
    const uint32_t frames = argc > 5 ? uint32_t(atoi(argv[5])) : 16, bounces = argc > 6 ? uint32_t(atoi(argv[6])) : 6;
    rtxpt_host_scene* scene = nullptr; uint32_t overridden = 0;
    const size_t len = strlen(argv[1]); const bool sceneFile = len > 11 && !strcmp(argv[1] + len - 11, ".scene.json");
    if (sceneFile ? rtxpt_b200_load_scene_json(argv[1], nullptr, &scene) != RTXPT_OK : rtxpt_b200_load_gltf_ex(argv[1], nullptr, nullptr, &scene, &overridden) != RTXPT_OK) return fail("load", nullptr);
    uint32_t cameraCount = 1; RtxptGltfCamera gcam = {};
    rtxpt_b200_host_scene_cameras(scene, &gcam, &cameraCount);
    if (cameraCount == 0) { fprintf(stderr, "the file has no perspective camera\n"); return 1; }
    RtxptCameraData cam; const float jitter[2] = { 0, 0 };
    rtxpt_b200_bridge_camera(width, height, gcam.position, gcam.direction, gcam.up, gcam.yfov, gcam.znear, gcam.zfar > 0 ? gcam.zfar : 1e7f, 10000.0f, 0.0f, jitter, &cam);
    float worldToView[16], viewToClip[16], worldToClip[16];
    rtxpt_b200_camera_matrices(&cam, worldToView, viewToClip, worldToClip);

    RtxptPathTracerConstants consts; rtxpt_b200_default_constants(&cam, 0, &consts);
    consts.bounceCount = bounces; consts.diffuseBounceCount = bounces < 3 ? bounces : 3;
    consts.NEEType = 2; consts.NEEATFeedback = 1; consts.NEEATImportanceBoost = 3;                     // RTXPT's defaults: NEE-AT with temporal feedback and both importance boosters
    consts.useApproximateMIS = approximateMIS ? 1u : 0u;                                              // pt.useApproximateMIS = m_ui.ActualUseApproximateMIS()
    RtxptRealtimeConstants rt = {};
    rt.activeStablePlaneCount = 3; rt.maxStablePlaneVertexDepth = bounces < 14 ? bounces : 14; rt.allowPrimarySurfaceReplacement = 1; rt.subSampleCount = 1;
    memcpy(rt.matWorldToClipNoOffset, worldToClip, 64); memcpy(rt.prevMatWorldToClipNoOffset, worldToClip, 64);
    rt.clipToWindowScale[0] = 0.5f * float(width); rt.clipToWindowScale[1] = -0.5f * float(height);
    RtxptDenoiserConstants dn = {};
    memcpy(dn.matWorldToView, worldToView, 64);
    dn.hitDistanceParameters[0] = 3.0f; dn.hitDistanceParameters[1] = 0.1f; dn.hitDistanceParameters[2] = 20.0f; dn.hitDistanceParameters[3] = -25.0f;   // nrd::HitDistanceParameters defaults
    dn.preExposedGrayLuminance = 1.0f; dn.denoiserRadianceClampK = 8.0f;
    RtxptReblurFrame rf = {};
    memcpy(rf.matWorldToView, worldToView, 64); memcpy(rf.matViewToClip, viewToClip, 64); memcpy(rf.prevMatWorldToView, worldToView, 64); memcpy(rf.prevMatViewToClip, viewToClip, 64);
    RtxptToneMappingParams tm = {};
    tm.toneMapOperator = 5; tm.clamped = 1; tm.enabled = 1; tm.autoExposure = 1; tm.exposureValueMin = -16.0f; tm.exposureValueMax = 16.0f; tm.whiteScale = 11.2f; tm.whiteMaxLuminance = 1.0f;
    tm.whitePoint = 6500.0f; tm.filmSpeed = 100.0f; tm.fNumber = 1.0f; tm.shutter = 1.0f;

    RtxptConfig cfg = {}; cfg.deviceOrdinal = -1; cfg.maxSubSamplesPerLaunch = 1; cfg.tileWorld = 1; cfg.tileSize = 64;
    rtxpt_ctx* ctx = nullptr;
    if (rtxpt_b200_create(&cfg, &ctx) != RTXPT_OK) return fail("create (a CUDA device is required; there is no CPU fallback)", ctx);
    TRY(rtxpt_b200_upload_scene(ctx, rtxpt_b200_host_scene_desc(scene)));
    rtxpt_b200_free_host_scene(scene);
    RtxptViewConstants view; memcpy(view.matWorldToClip, worldToClip, 64);
    float denoiseMs = 0;
    for (uint32_t f = 0; f < frames; f++)
    {
        consts.sampleBaseIndex = f;                                     // m_sampleIndex * ActualSamplesPerPixel()
        TRY(rtxpt_b200_set_constants(ctx, &consts));
        TRY(rtxpt_b200_set_view(ctx, &view));
        TRY(rtxpt_b200_set_realtime(ctx, &rt));
        TRY(rtxpt_b200_neeat_update_begin(ctx, nullptr));               // LightsBaker::UpdateBegin's feedback half
        TRY(rtxpt_b200_path_trace_realtime(ctx, 0, nullptr));           // BUILD, LightsBaker::UpdateEnd's passes, FILL
        rf.frameIndex = f; rf.resetHistory = f == 0;
        TRY(rtxpt_b200_denoise_realtime(ctx, &dn, &rf, nullptr));       // Sample::Denoise with ReBLUR
        TRY(rtxpt_b200_tone_map(ctx, &tm, RTXPT_BUFFER_OUTPUT_COLOR_F16, nullptr));
        rtxpt_b200_last_denoise_ms(ctx, &denoiseMs);
    }
    std::vector<unsigned char> ldr(size_t(width) * height * 4);
    TRY(rtxpt_b200_readback(ctx, RTXPT_BUFFER_LDR_COLOR_RGBA8, ldr.data(), ldr.size()));
    RtxptStats st; rtxpt_b200_get_stats(ctx, &st);
    fprintf(stderr, "%u x %u, %u frames, trace %.2f ms + denoise %.2f ms per frame (last)\n", width, height, frames, st.msTotal, denoiseMs);
    rtxpt_b200_destroy(ctx);
    FILE* out = fopen(argv[2], "wb"); if (!out) { perror(argv[2]); return 1; }
    fprintf(out, "P6\n%u %u\n255\n", width, height);
    for (size_t i = 0; i < size_t(width) * height; i++) fwrite(&ldr[i * 4], 1, 3, out);
    fclose(out);
    return 0;
}
