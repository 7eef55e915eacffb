"""ORACLE — TEST INFRASTRUCTURE.  Writes the sources of liboracle_amis.so (amis.mk): the oracle with RtxptPathTracerConstants::useApproximateMIS honoured.

The committed oracle (pt_path.h, oracle.cpp) is the full-MIS yardstick and stays as it is.  This script streams those two files into OUTDIR with the switch added where RTXPT's
shaders have their `#if RTXPT_USE_APPROXIMATE_MIS` arms - the light sample (PathTracerNEE.hlsli:228-232), the environment miss (PathTracer.hlsli:461-466), the emissive triangle
(:619-623, which then tests no light index) and the analytic-light proxy (LightSampler.hlsli:380-382) - plus pt_amis.h's two weights, and oracle_hit_funcs reading the switch from
word 94 of a "hit" record (tests/golden/hit_golden_amis.npz).  Every rewrite is an insertion in front of an unchanged line or expression, so with the switch at 0 the library
computes what liboracle.so computes; each anchor must occur exactly once, or the script fails.  The other headers are included from oracle/ as they are.

    python3 amis_oracle.py OUTDIR
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

PT_PATH = [
    # the two approximate weights, after EvalMISBalance / LightSample and before the firefly filter
    ("// ---- firefly filter (PathTracerHelpers.hlsli:183-219)",
     '#include "pt_amis.h"\n// ---- firefly filter (PathTracerHelpers.hlsli:183-219)'),
    # HandleMiss: no quad-tree lookup
    ("        if (misInfo.LightSamplingEnabled && bsdfScatterPdf != 0)\n",
     "        if (x.c->useApproximateMIS && misInfo.LightSamplingEnabled && bsdfScatterPdf != 0)\n"
     "            misWeight = ComputeLightVsBSDF_MIS_ForBSDF_Approx(bsdfScatterPdf, misInfo.CandidateSamples, misInfo.FullSamples);\n"
     "        else if (misInfo.LightSamplingEnabled && bsdfScatterPdf != 0)\n"),
    # HandleNEE: the light side
    ("            float pathMIS = ComputeLightVsBSDF_MIS_ForLight(picked, thisPdf, otherPdf, fullSamples, scatterPdfForDir);",
     "            float pathMIS = x.c->useApproximateMIS ? ComputeLightVsBSDF_MIS_ForLight_Approx(picked, candidateSampleCount, fullSamples, scatterPdfForDir)\n"
     "                                                   : ComputeLightVsBSDF_MIS_ForLight(picked, thisPdf, otherPdf, fullSamples, scatterPdfForDir);"),
    # HandleHitSurface, emissive triangle: weighted with or without a light record
    ("        if (misInfo.LightSamplingEnabled && bsdfScatterPdf != 0 && surface.neeTriangleLightIndex != RTXPT_INVALID_LIGHT_INDEX)\n",
     "        if (x.c->useApproximateMIS && misInfo.LightSamplingEnabled && bsdfScatterPdf != 0)\n"
     "            misWeight = ComputeLightVsBSDF_MIS_ForBSDF_Approx(bsdfScatterPdf, misInfo.CandidateSamples, misInfo.FullSamples);\n"
     "        else if (misInfo.LightSamplingEnabled && bsdfScatterPdf != 0 && surface.neeTriangleLightIndex != RTXPT_INVALID_LIGHT_INDEX)\n"),
    # analytic-light proxy
    ("                if (bsdfPdf != 0) mis = ComputeLightVsBSDF_MIS_ForBSDF(",
     "                if (bsdfPdf != 0 && x.c->useApproximateMIS) mis = ComputeLightVsBSDF_MIS_ForBSDF_Approx(bsdfPdf, misInfo.CandidateSamples, misInfo.FullSamples);\n"
     "                else if (bsdfPdf != 0) mis = ComputeLightVsBSDF_MIS_ForBSDF("),
]
ORACLE_CPP = [
    ("c.EnvironmentMapDiffuseSampleMIPLevel = r[93]; c.NEEATFeedback = 1;",
     "c.EnvironmentMapDiffuseSampleMIPLevel = r[93]; c.NEEATFeedback = 1; c.useApproximateMIS = uint(r[94]);"),
]


def rewrite(name, edits, out):
    with open(os.path.join(HERE, name)) as f:
        text = f.read()
    for old, new in edits:
        n = text.count(old)
        if n != 1:
            sys.exit("amis_oracle.py: %s: anchor found %d times (expected once): %r" % (name, n, old[:80]))
        text = text.replace(old, new)
    with open(os.path.join(out, name), "w") as f:
        f.write(text)


if __name__ == "__main__":
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    rewrite("pt_path.h", PT_PATH, out)
    rewrite("oracle.cpp", ORACLE_CPP, out)
