// ORACLE — TEST INFRASTRUCTURE.  Approximate light-vs-BSDF MIS (RTXPT_USE_APPROXIMATE_MIS = 1, RtxptPathTracerConstants::useApproximateMIS): LightSampler::
// ComputeLightVsBSDF_MIS_ForLight_Approx / _ForBSDF_Approx (Lighting/LightSampler.hlsli:271-280).  The light's selection x solid-angle pdf is the constant
// RTXPT_NEEAT_MIS_APPROXIMATION_LIGHTSAMPLER_BIAS; the BSDF side needs no light index, record or sampler pdf.
// Not included by the full-MIS oracle: amis_oracle.py places it in pt_path.h for liboracle_amis.so (amis.mk), after EvalMISBalance and LightSample.
constexpr float kApproxMISLightSamplerBias = 3.0f;
inline float ComputeLightVsBSDF_MIS_ForLight_Approx(const LightSample& s, uint candidateSampleCount, uint fullSampleCount, float bsdfPdf)
{
    return EvalMISBalance(float(fullSampleCount * candidateSampleCount), kApproxMISLightSamplerBias, 1, s.LightSampleableByBSDF ? bsdfPdf : 0.0f);
}
inline float ComputeLightVsBSDF_MIS_ForBSDF_Approx(float bsdfPdf, uint candidateSampleCount, uint fullSampleCount)
{
    return EvalMISBalance(1, bsdfPdf, float(fullSampleCount * candidateSampleCount), kApproxMISLightSamplerBias);
}
