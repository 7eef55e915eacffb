// ORACLE build with RTXPT's DLSS-RR input pass — test infrastructure only.  The committed oracle (oracle.cpp, unchanged) plus two entries over pt_dlss_rr.h:
//   oracle_dlss_rr_records  the pass on single pixels given record by record (the layout of ref_kat_dlss_rr, tests/golden/make_dlss_rr_golden.py): 104 words in, 15 floats out
//   oracle_dlss_rr_frame    the pass over a whole frame's realtime targets (a context's own buffers), written in the targets' formats
#include "oracle.cpp"
#include "pt_dlss_rr.h"

extern "C" {

ORC_API void oracle_dlss_rr_records(const uint32_t* in, uint32_t count, float* out)
{
    RtxptRealtimeConstants rt{};
    RtxptStablePlane planes[3 * 64]; uint32_t header[4]; uint16_t stableRadiance[4], motion[4]; float specHitT;
    RealtimeTargets T; T.width = T.height = 1; T.lineStride = GenericTSComputeLineStride(1, 1); T.planeStride = GenericTSComputePlaneStride(1, 1);
    T.planes = planes; T.header = header; T.stableRadiance = stableRadiance; T.motionVectors = motion; T.specularHitT = &specHitT; T.rt = &rt;
    for (uint32_t i = 0; i < count; i++, in += 104, out += 15)
    {
        rt.activeStablePlaneCount = in[0];
        const float clampK = asfloat(in[1]);
        memcpy(header, in + 2, 16);
        memset(planes, 0, sizeof(planes));
        for (uint k = 0; k < 3; k++) memcpy(&planes[T.PixelToAddress(0, 0, k)], in + 6 + 20 * k, 80);
        memcpy(stableRadiance, in + 66, 8); memcpy(&specHitT, in + 68, 4); memcpy(motion, in + 69, 4); motion[2] = motion[3] = 0;
        dlssrr::View v; v.worldToClip = reinterpret_cast<const float*>(in + 70); v.prevWorldToClip = reinterpret_cast<const float*>(in + 86);
        v.clipToWindowScale[0] = asfloat(in[102]); v.clipToWindowScale[1] = asfloat(in[103]);
        const dlssrr::Result R = dlssrr::pixel(T, v, clampK, 0, 0);
        const float o[15] = { R.color.x, R.color.y, R.color.z, R.diffAlbedo.x, R.diffAlbedo.y, R.diffAlbedo.z, R.specAlbedo.x, R.specAlbedo.y, R.specAlbedo.z,
                              R.normal.x, R.normal.y, R.normal.z, R.roughness, R.specMotion.x, R.specMotion.y };
        memcpy(out, o, sizeof(o));
    }
}

// realtimeTargets: planes, header, stable radiance, depth, motion vectors (RGBA16F), throughput, specular hit distance - as oracle_denoiser_prepare_inputs takes them;
// outputs: colour RGBA16F, diffuse / specular albedo R11G11B10, normals + roughness RGBA16F, specular motion vectors RG16F (full frame, row-major)
ORC_API int oracle_dlss_rr_frame(uint32_t W, uint32_t H, const RtxptRealtimeConstants* rt, float brightnessClampK, void* const* r, uint16_t* outColor, uint32_t* outDiffAlbedo,
                                 uint32_t* outSpecAlbedo, uint16_t* outNormalsRoughness, uint16_t* outSpecMotion)
{
    if (!rt || !r || W == 0 || H == 0) return -1;
    RealtimeTargets T; T.width = W; T.height = H; T.lineStride = GenericTSComputeLineStride(W, H); T.planeStride = GenericTSComputePlaneStride(W, H);
    T.planes = (RtxptStablePlane*)r[0]; T.header = (uint32_t*)r[1]; T.stableRadiance = (uint16_t*)r[2]; T.depth = (float*)r[3]; T.motionVectors = (uint16_t*)r[4]; T.throughput = (uint32_t*)r[5];
    T.specularHitT = (float*)r[6]; T.rt = rt;
    dlssrr::View v; v.worldToClip = rt->matWorldToClipNoOffset; v.prevWorldToClip = rt->prevMatWorldToClipNoOffset; v.clipToWindowScale[0] = rt->clipToWindowScale[0]; v.clipToWindowScale[1] = rt->clipToWindowScale[1];
    const dlssrr::Targets O{ outColor, outDiffAlbedo, outSpecAlbedo, outNormalsRoughness, outSpecMotion };
    #pragma omp parallel for schedule(dynamic, 4)
    for (int y = 0; y < int(H); y++) for (uint32_t x = 0; x < W; x++) dlssrr::store(T, O, dlssrr::pixel(T, v, brightnessClampK, x, uint32_t(y)), x, uint32_t(y));
    return 0;
}

} // extern "C"
