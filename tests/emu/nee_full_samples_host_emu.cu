// TEST INFRASTRUCTURE ONLY - never linked into librtxpt_b200*.so.  Host build of the multi-sample shade (NEEFullSamples > 1): shade.cuh's shadeHit< .., MULTI > - what
// k_shade< .., MULTI > (reference mode) and k_rt_shade< FILL, .., MULTI > run per vertex - followed by what k_trace_shadow< .., MULTI > and k_nee_resolve do with the vertex's shadow
// records and NEE block, on records of tests/golden/hit_golden.npz, for tests/test_nee_full_samples_port.py.  The device-only spellings, the stub bridge's hooks (surface,
// environment cube, camera) and its visibility rule are those of shade_host_emu.cu, included here; this library is built on its own (nee_full_samples.mk).
#include "shade_host_emu.cu"

// One path vertex, set up from the record as shadeVertex (shade_host_emu.cu) sets it up, shaded with NEEFullSamples light samples and no feedback insertion.  Every sample's shadow
// ray gets the stub's visibility answer, then the block is resolved - in reverse sample order with `reverseSum`, to show that the order matters.  Outputs as shadeVertex: the
// path state, the number of shadow rays (20), the last sample's ray and answer (21-28), planes / header / stable radiance (realtime), the feedback reservoir.  Returns 0, or -1 for
// a record this path does not cover (ops other than hit and miss, feedback insertion).
template <int MODE> static int shadeVertexMulti(const float* r, float* o, bool reverseSum)
{
    constexpr bool kRealtime = MODE != kModeReference, kNeeat = MODE != kModeBuildStablePlanes;     // k_shade< .., NEEAT >, k_rt_shade< BUILD, .. >, k_rt_shade< FILL, .., NEEAT >
    for (int k = 0; k < 128; k++) o[k] = 0.0f;
    if (r[27] > 1.0f) return -1;
    if (r[92] != 0.0f) return -1;         // feedback insertion with several samples: refused by rtxpt_b200_set_constants
    LaunchParams p; memset(&p, 0, sizeof(p));
    // surface
    Surface s; memset(&s, 0, sizeof(s));
    s.posW = mk3(r[28], r[29], r[30]); s.faceN = mk3(r[31], r[32], r[33]); s.V = mk3(-r[23], -r[24], -r[25]); s.N = mk3(r[34], r[35], r[36]); s.T = mk3(r[37], r[38], r[39]); s.B = mk3(r[40], r[41], r[42]);
    s.vertexN = mk3(r[43], r[44], r[45]); s.frontFacing = r[46] != 0.0f; s.nestedPriority = uint(r[47]); s.thin = r[49] != 0.0f; s.psdExclude = r[50] != 0.0f; s.materialID = uint(r[51]); s.IoR = r[52];
    s.shadowNoLFadeout = r[53]; s.emission = mk3(r[54], r[55], r[56]); s.psdBlockMVs = r[57] != 0.0f; s.psdDominantDeltaLobeP1 = uint(r[58]);
    const float* b = r + 42;
    s.bsdf.diffuse = mk3(b[18], b[19], b[20]); s.bsdf.roughness = b[21]; s.bsdf.specular = mk3(b[22], b[23], b[24]); s.bsdf.metallic = b[25]; s.bsdf.transmission = mk3(b[26], b[27], b[28]);
    s.bsdf.diffuseTransmission = b[29]; s.bsdf.specularTransmission = b[30]; s.bsdf.eta = b[31];
    s.interiorIoR = r[74]; s.neeTriangleLightIndex = r[75] < 0 ? 0xFFFFFFFFu : uint(r[75]); s.neeAnalyticLightIndex = r[76] < 0 ? 0xFFFFFFFFu : uint(r[76]); s.prevPosW = mk3(r[77], r[78], r[79]);
    gSurface = &s;
    // constants
    RtxptPathTracerConstants& c = p.c;
    c.imageWidth = c.imageHeight = 8; c.bounceCount = uint(r[80]); c.diffuseBounceCount = uint(r[81]); c.NEEEnabled = 1; c.NEEType = 2; c.NEECandidateSamples = uint(r[83]); c.NEEFullSamples = uint(r[84]);
    c.fireflyFilterThreshold = r[85]; c.enableRussianRoulette = 1; c.enableLDSamplerForBSDF = 1; c.nestedDielectricsQuality = 1; c.EnvironmentMapDiffuseSampleMIPLevel = r[93]; c.NEEATFeedback = 1;
    for (int a = 0; a < 3; a++) for (int k = 0; k < 3; k++) { c.envMap.Transform[a * 4 + k] = r[950 + 3 * a + k]; c.envMap.InvTransform[k * 4 + a] = r[950 + 3 * a + k]; }
    for (int k = 0; k < 3; k++) c.envMap.ColorMultiplier[k] = r[959];
    // scene side: materials, lights
    RtxptMaterialData mats[8]; memset(mats, 0, sizeof(mats));
    for (int m = 0; m < 8; m++) { mats[m].IoR = r[96 + m]; for (int k = 0; k < 3; k++) mats[m].VolumeAttenuationColor[k] = r[104 + 3 * m + k]; mats[m].VolumeAttenuationDistance = r[128 + m]; }
    p.scene.materials = mats; p.scene.materialCount = 8;
    LightInfo lights[16]; uint4 lightsEx[16]; uint32_t counters[16], indices[64], local[512], proxyCount = uint(r[90]);
    for (int k = 0; k < 16; k++) { memcpy(&lights[k], r + 728 + 12 * k, 32); memcpy(&lightsEx[k], r + 728 + 12 * k + 8, 16); counters[k] = uint(r[136 + k]); }
    for (int k = 0; k < 64; k++) indices[k] = uint(r[152 + k]);
    memcpy(local, r + 216, sizeof(local));
    p.scene.lights = lights; p.scene.lightCount = 16; p.scene.analyticLightCount = 16; p.scene.envEnabled = 1; p.scene.envLookupMap = envLookup().data();
    // shade.cuh reads the Extended record of light i at lightsEx[ uint( i - 5368 ) ] (the analytic lights follow the 5368 environment nodes): make that land on entry i of this 16-light table
    p.scene.lightsEx = reinterpret_cast<const uint4*>(reinterpret_cast<uintptr_t>(lightsEx) - (uintptr_t(0x100000000ull) - 5368ull) * sizeof(uint4));
    p.scene.proxyCounters = counters; p.scene.proxyIndices = indices; p.scene.samplingProxyCount = proxyCount;
    float fbWeight[64]; uint32_t fbCand[64]; for (int k = 0; k < 64; k++) { fbWeight[k] = 0.0f; fbCand[k] = 0xFFFFFFFFu; }
    p.na.W = p.na.H = 8; p.na.tilesX = p.na.tilesY = 2; p.na.lightCount = 16; p.na.neeType = 2; p.na.jitterX = uint(r[88]); p.na.jitterY = uint(r[89]); p.na.localToGlobalSampleRatio = r[86];
    p.na.screenSpaceVsWorldSpaceThreshold = r[91]; p.na.temporalFeedbackRequired = uint(r[92]); p.na.fbWeight = fbWeight; p.na.fbCandidate = fbCand; p.na.localSamplingBuffer = local;
    p.na.proxyCounters = counters; p.na.proxyIndices = indices; p.na.samplingProxyCount = &proxyCount;
    uint32_t rrFix[1] = { 0u }; p.naRrFix = rrFix;
    // realtime passes: the stable planes of an 8 x 8 image, the pixel's entries from the record; the stub bridge's camera
    const uint32_t pid = emu::f2u(r[3]), px = (pid >> 16) & 7u, py = pid & 7u;
    RtxptStablePlane planes[3 * 64]; uint32_t header[4 * 64]; uint2 stableRadiance[64]; float specHitT[64], depth[64]; uint2 motion[64]; uint32_t throughput[64];
    if (kRealtime)
    {
        memset(planes, 0, sizeof(planes)); memset(header, 0xFF, sizeof(header)); memset(stableRadiance, 0, sizeof(stableRadiance)); memset(motion, 0, sizeof(motion)); memset(throughput, 0, sizeof(throughput));
        for (int k = 0; k < 64; k++) { specHitT[k] = 0.0f; depth[k] = -1.0f; }
        p.rt.planes = planes; p.rt.header = header; p.rt.stableRadiance = stableRadiance; p.rt.specularHitT = specHitT; p.rt.lineStride = 8; p.rt.planeStride = 64; p.rt.activePlaneCount = 3;
        p.rt.maxVertexDepth = uint(r[943]); p.rt.allowPSR = uint(r[944]); p.rt.attenuation = r[87]; p.depth = depth; p.motionVectors = motion; p.throughput = throughput;
        for (int k = 0; k < 16; k += 5) p.worldToClip[k] = 1.0f;
        for (uint32_t k = 0; k < 4; k++) memcpy(&header[(k * 8 + py) * 8 + px], r + 920 + k, 4);
        for (uint32_t k = 0; k < 3; k++) memcpy(planes[planeAddress(p.rt, (px << 16) | py, k)].PackedNoisyRadianceAndSpecAvg, r + 924 + 2 * k, 8);
        specHitT[py * 8 + px] = r[930];
        stableRadiance[py * 8 + px] = make_uint2(f32tof16(r[946]) | (f32tof16(r[947]) << 16), f32tof16(r[948]) | (f32tof16(r[949]) << 16));
        gCamPos = mk3(r[931], r[932], r[933]); gCamBase = mk3(r[934], r[935], r[936]); gCamDx = mk3(r[937], r[938], r[939]); gCamDy = mk3(r[940], r[941], r[942]);
        p.firstSampleIndex = uint(r[82]);
    }
    // the path: the 80-byte payload in the order of wavefront.cuh's five state words (the stableBranchID word carries the sample index in reference mode)
    uint32_t w[20]; memcpy(w, r, 80);
    PathRegs path;
    path.origin = mk3(emu::u2f(w[0]), emu::u2f(w[1]), emu::u2f(w[2])); path.id = w[3]; path.dir = mk3(emu::u2f(w[4]), emu::u2f(w[5]), emu::u2f(w[6])); path.sceneLength = emu::u2f(w[7]);
    path.thpXY = w[8]; path.thpZ = w[9]; path.lXY = w[10]; path.lZW = w[11]; path.interior0 = w[12]; path.interior1 = w[13]; path.packedCounters = w[14]; path.rayCone = w[16];
    path.pack0 = w[17]; path.pack1 = w[18]; path.flagsAndVertexIndex = w[19]; path.sampleIndex = kRealtime ? w[15] : uint(r[82]);
    HitOutputs out; out.continuePath = false; out.emitShadow = false; out.naRecord = make_uint4(0xFFFFFFFFu, 0u, 0u, 0u);
    // the launch arrays of one path - a counter block, N shadow records, one NEE block; the path's L where k_nee_resolve finds it (radiance[h] / s2 of the slot)
    const uint32_t fullSamples = min(kNeeMaxFullSamples, c.NEEFullSamples);
    uint32_t ctr[kCountersPerIter] = {}; float4 recOriginTMax[kNeeMaxFullSamples], recDirPath[kNeeMaxFullSamples]; uint2 recSample[kNeeMaxFullSamples];
    uint4 block[1 + kNeeMaxFullSamples]; uint2 radianceWord[1]; uint4 s2Word[1];
    p.wf.counters = ctr; p.wf.capacity = 1; p.iteration = 0; p.shadowLongRayT = 3.0e38f;
    p.wf.shadowOriginTMax = recOriginTMax; p.wf.shadowDirPath = recDirPath; p.wf.shadowRadiance = recSample; p.neeBlocks = block;
    p.radiance = radianceWord; p.wf.s2 = s2Word;
    if (r[27] == 1.0f) shadeMiss<false, MODE, kNeeat>(p, path);
    else shadeHit<false, true, MODE, kNeeat, true>(p, path, 0u, make_float4(r[26], 0.25f, 0.25f, 0.0f), out);
    if (ctr[kCtrNeeBlocks] != 0)
    {   // k_trace_shadow< .., MULTI >: every record's visibility marks its sample (records are kept in the order they were appended: back to front); the last sample's ray is reported
        const uint32_t records = ctr[kCtrShadowCount] + ctr[kCtrShadowShort], capacity = neeShadowCapacity(p);
        uint32_t lastSample = 0;
        for (uint32_t i = 0; i < records; i++)
        {
            const uint32_t e = shadowRecordIndex(i, ctr[kCtrShadowCount], capacity), j = recSample[e].x;
            const bool visible = visibilityRule(recOriginTMax[e], recDirPath[e]);
            if (visible) { if (j < 32) block[0].z |= 1u << j; else block[0].w |= 1u << (j - 32); }
            if (i == 0 || j >= lastSample)
            {
                lastSample = j;
                o[21] = recOriginTMax[e].x; o[22] = recOriginTMax[e].y; o[23] = recOriginTMax[e].z; o[24] = recDirPath[e].x; o[25] = recDirPath[e].y; o[26] = recDirPath[e].z;
                o[27] = recOriginTMax[e].w; o[28] = visible ? 1.0f : 0.0f;
            }
        }
        o[20] = float(records);
        // k_nee_resolve
        radianceWord[0] = make_uint2(path.lXY, path.lZW); s2Word[0] = make_uint4(0u, 0u, path.lXY, path.lZW);
        if (!reverseSum) resolveNeeBlock<kRealtime>(p, block);
        else
        {
            uint2 sum = make_uint2(0u, 0u);
            for (int j = int(fullSamples) - 1; j >= 0; j--)
                if ((j < 32 ? block[0].z >> j : block[0].w >> (j - 32)) & 1u)
                {
                    const uint4 s = block[1 + j];
                    sum.x = packHalf2Clamp(f16tof32(sum.x) + emu::u2f(s.x), f16tof32(sum.x >> 16) + emu::u2f(s.y));
                    sum.y = packHalf2Clamp(f16tof32(sum.y) + emu::u2f(s.z), f16tof32(sum.y >> 16) + emu::u2f(s.w));
                }
            sum.x |= block[0].y;
            accumulateNeeRadiance<kRealtime>(p, 0u, sum);
        }
        if (kRealtime) { path.lXY = s2Word[0].z; path.lZW = s2Word[0].w; } else { path.lXY = radianceWord[0].x; path.lZW = radianceWord[0].y; }
    }
    // the outgoing path state (as shadeVertex reports it) and the pixel's feedback reservoir (empty: no insertion without temporalFeedbackRequired)
    uint32_t q[20] = { emu::f2u(path.origin.x), emu::f2u(path.origin.y), emu::f2u(path.origin.z), path.id, emu::f2u(path.dir.x), emu::f2u(path.dir.y), emu::f2u(path.dir.z), emu::f2u(path.sceneLength),
                       path.thpXY, path.thpZ, path.lXY, path.lZW, path.interior0, path.interior1, path.packedCounters, kRealtime ? path.sampleIndex : w[15], path.rayCone, path.pack0, path.pack1, path.flagsAndVertexIndex };
    memcpy(o, q, 80);
    if (kRealtime)
    {
        o[37] = specHitT[py * 8 + px];
        for (uint32_t k = 0; k < 3; k++) { const RtxptStablePlane& sp = planes[planeAddress(p.rt, (px << 16) | py, k)]; memcpy(o + 41 + 2 * k, sp.PackedNoisyRadianceAndSpecAvg, 8); memcpy(o + 56 + 20 * k, &sp, 80); }
        for (uint32_t k = 0; k < 4; k++) memcpy(o + 47 + k, &header[(k * 8 + py) * 8 + px], 4);
        const uint2 sr = stableRadiance[py * 8 + px]; o[52] = f16tof32(sr.x); o[53] = f16tof32(sr.x >> 16); o[54] = f16tof32(sr.y); o[55] = f16tof32(sr.y >> 16);
    }
    const uint32_t at = (path.id & 7u) * 8 + ((path.id >> 16) & 7u);
    o[39] = fbWeight[at]; memcpy(o + 40, &fbCand[at], 4);
    return 0;
}

// `count` records of 1024 floats, 128 floats out each; mode 0 = reference, 2 = FILL; status[i] = 0 where the record was run
extern "C" void nee_emu_multi_vertices(const float* in, uint32_t count, float* out, int32_t* status, uint32_t mode, int32_t reverseSum)
{
    for (uint32_t i = 0; i < count; i++)
    {
        const float* r = in + size_t(i) * 1024; float* o = out + size_t(i) * 128;
        status[i] = mode == 0 ? shadeVertexMulti<kModeReference>(r, o, reverseSum != 0) : (mode == 2 ? shadeVertexMulti<kModeFillStablePlanes>(r, o, reverseSum != 0) : -1);
    }
}
