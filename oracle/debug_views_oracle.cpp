// ORACLE build with RTXPT's debug views — test infrastructure only.  The committed oracle (oracle.cpp, unchanged) plus two entries:
//   oracle_debug_first_hit     surfaceDebugViz at path vertex 1: the camera ray of (pixel, sampleIndex), its closest hit, Bridge::loadSurface there exactly as HandleHit
//                              calls it (UpdatePathTravelled first, so the ray cone has travelled the hit distance), then the view's colour
//   oracle_debug_stable_planes StablePlanesDebugViz over the plane buffers oracle_render_realtime filled
// Both write RGBA32F per pixel (row-major, full image); pixels where nothing is drawn keep 0, the cleared debug target.
#include "oracle.cpp"
#include "pt_debug_views.h"

extern "C" {

ORC_API int oracle_debug_first_hit(void* p, uint32_t view, uint32_t sampleIndex, float* outRGBA, int threads)
{
    OracleCtx* c = (OracleCtx*)p;
    if (!c->haveConsts || !outRGBA) return -1;
    const uint32_t W = c->consts.imageWidth, H = c->consts.imageHeight;
#ifdef _OPENMP
    if (threads > 0) omp_set_num_threads(threads);
#endif
    #pragma omp parallel
    {
        PathTracerCtx x; x.scene = &c->scene; x.bvh = &c->bvh; x.lights = &c->lights; x.c = &c->consts; x.stats = nullptr; x.sampleIndex = sampleIndex;
        #pragma omp for schedule(dynamic, 1)
        for (int y = 0; y < int(H); y++)
            for (uint32_t px = 0; px < W; px++)
            {
                float* o = outRGBA + (size_t(y) * W + px) * 4; o[0] = o[1] = o[2] = o[3] = 0.0f;
                PathState path = EmptyPathInitialize(x, px, uint32_t(y), c->consts.camera.PixelConeSpreadAngle);
                computeCameraRay(x, px, uint32_t(y), path.origin, path.dir);
                const Hit h = c->bvh.trace(c->scene, path.origin, path.dir, 0.0f, kMaxRayTravel, false);
                if (!h.valid()) continue;
                UpdatePathTravelled(path, h.t);
                const Tri& tri = c->bvh.tris[h.triId];
                const SurfaceData s = loadSurface(c->scene, tri.instanceIndex, tri.geometryIndex, tri.primitiveIndex, f2(h.u, h.v), path.dir, path.rayCone, c->consts.texLODBias,
                                                  path.getVertexIndex(), path.id >> 16, path.id & 0xFFFF, sampleIndex);
                const float4 v = dbgviz::SurfaceDebugViz(view, s, f2(h.u, h.v));
                o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
            }
    }
    return 0;
}

// realtimeTargets as for oracle_denoiser_prepare_inputs; dbgPlaneIndex: 0..2, or -1 for the four-way split (RTXPT's debugViewStablePlaneIndex)
ORC_API int oracle_debug_stable_planes(void* p, const RtxptRealtimeConstants* rt, uint32_t view, int32_t dbgPlaneIndex, void* const* realtimeTargets, float* outRGBA)
{
    OracleCtx* c = (OracleCtx*)p;
    if (!c->haveConsts || !rt || !outRGBA) return -1;
    const RealtimeTargets T = makeTargets(c, rt, realtimeTargets);
    for (uint32_t y = 0; y < T.height; y++)
        for (uint32_t px = 0; px < T.width; px++)
        {
            const float4 v = dbgviz::StablePlanesDebugViz(T, view, dbgPlaneIndex, px, y);
            float* o = outRGBA + (size_t(y) * T.width + px) * 4;
            if (v.w > 0) { o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w; } else { o[0] = o[1] = o[2] = o[3] = 0.0f; }
        }
    return 0;
}

// surfaceDebugViz on a surface given field by field: per record 28 words - barycentrics (2), faceNCorrected, vertexN, N, T, B (15), frontFacing, isThinSurface, diffuse (3),
// specular (3), roughness, metallic (f32), materialID (u32) -> 4 floats
ORC_API void oracle_debug_first_hit_records(uint32_t view, const uint32_t* in, uint32_t count, float* out)
{
    for (uint32_t i = 0; i < count; i++, in += 28)
    {
        SurfaceData s = {}; ShadingData& sd = s.sd; StandardBSDFData& b = s.bsdf.data;
        float3* v[5] = { &sd.faceNCorrected, &sd.vertexN, &sd.N, &sd.T, &sd.B };
        for (int k = 0; k < 5; k++) *v[k] = f3(asfloat(in[2 + 3 * k]), asfloat(in[3 + 3 * k]), asfloat(in[4 + 3 * k]));
        sd.frontFacing = in[17] != 0; sd.thinSurface = in[18] != 0;
        b.diffuse = f3(asfloat(in[19]), asfloat(in[20]), asfloat(in[21])); b.specular = f3(asfloat(in[22]), asfloat(in[23]), asfloat(in[24]));
        b.roughness = asfloat(in[25]); b.metallic = asfloat(in[26]); sd.materialID = in[27];
        const float4 c = dbgviz::SurfaceDebugViz(view, s, f2(asfloat(in[0]), asfloat(in[1])));
        out[4 * i] = c.x; out[4 * i + 1] = c.y; out[4 * i + 2] = c.z; out[4 * i + 3] = c.w;
    }
}

// the final merge's debug views for one plane (realtimeTargets / denoiserTargets as for oracle_denoiser_final_merge), drawn into outRGBA, which keeps what earlier merges drew
ORC_API int oracle_debug_denoiser_merge(void* p, const RtxptRealtimeConstants* rt, uint32_t stablePlaneIndex, int32_t dbgPlaneIndex, uint32_t view, void* const* realtimeTargets,
                                        void* const* denoiserTargets, const uint16_t* denoisedDiff, const uint16_t* denoisedSpec, float* outRGBA)
{
    OracleCtx* c = (OracleCtx*)p;
    if (!c->haveConsts || !rt || stablePlaneIndex >= 3 || !outRGBA) return -1;
    const RealtimeTargets T = makeTargets(c, rt, realtimeTargets); const DenoiserTargets D = makeDenoiserTargets(denoiserTargets);
    dbgviz::DenoiserFinalMergeDebugViz(T, D, stablePlaneIndex, dbgPlaneIndex, view, denoisedDiff, denoisedSpec, outRGBA);
    return 0;
}

// the colour functions alone, in the records of oracle/ref_kat_debug_main.cpp (tests/golden/debug_view_golden.npz): per record op, a, b, c -> 3 words
ORC_API void oracle_debug_pixel_funcs(const uint32_t* in, uint32_t count, uint32_t* out)
{
    for (uint32_t i = 0; i < count; i++, in += 4, out += 3)
    {
        const uint32_t op = in[0], a = in[1], b = in[2], c = in[3];
        if (op == 3)
        {
            uint r[3]; dbgviz::StablePlaneDebugVizFourWaySplitCoord(int(a), b & 0xFFFFu, b >> 16, c & 0xFFFFu, c >> 16, r);
            out[0] = r[0]; out[1] = r[1]; out[2] = r[2];
            continue;
        }
        float3 r;
        if (op == 0) r = dbgviz::ColorFromHash(a);
        else if (op == 1) r = dbgviz::GradientHeatMap(asfloat(a));
        else if (op == 2) r = dbgviz::StablePlaneDebugVizColor(a);
        else r = dbgviz::DbgShowNormalSRGB(f3(asfloat(a), asfloat(b), asfloat(c)));
        out[0] = asuint(r.x); out[1] = asuint(r.y); out[2] = asuint(r.z);
    }
}

} // extern "C"
