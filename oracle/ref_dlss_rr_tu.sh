#!/usr/bin/env bash
# ORACLE/_ref — TEST INFRASTRUCTURE.  Writes ONE C++ translation unit to stdout for ref_kat_dlss_rr_main.cpp: the translation unit of ref_hlsl_tu.sh (shim, the UNMODIFIED path-tracer
# headers) with ref_kat_dlss_rr_main.cpp's stand-ins as its tail, then ProcessingPasses/PostProcess.hlsl:94-160 (ComputeSpecularMotionVector) and :175-440 (the DENOISER_DLSS_RR
# pass) of the UNMODIFIED reference read from where they lie under $REF, through ref_hlsl_tu.sh's spelling filter plus three rewrites of this file's own:
#   [numthreads(..)] and the SV_DispatchThreadID semantic     dropped; the entry point is named DlssRrPrepareInputsMain
#   1e-3 (literal with an exponent and no point)             -> 1e-3f: an HLSL literal takes the binary32 type of the expression it meets (the filter's rule for 1.5 -> 1.5f)
#   RTXPT_ACTIVE_STABLE_PLANE_COUNT                          a variable the driver sets per record, instead of ref_hlsl_tu.sh's 3
# then the driver.  Nothing of the reference is written to disk.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
eval "$(sed -n '/^filter() {/,/^}/p' "$HERE/ref_hlsl_tu.sh")"
PP=$REF/Rtxpt/ProcessingPasses/PostProcess.hlsl
REF=$REF "$HERE/ref_hlsl_tu.sh" "$HERE/ref_kat_dlss_rr_main.cpp" | sed -E 's/^#define RTXPT_ACTIVE_STABLE_PLANE_COUNT 3$/static uint g_shimActivePlaneCount = 3;\n#define RTXPT_ACTIVE_STABLE_PLANE_COUNT g_shimActivePlaneCount/'
pass() {
  sed -E -e 's/^[[:space:]]*\[numthreads\(.*\)\][[:space:]]*$//' \
         -e 's/void main\( uint3 dispatchThreadID : SV_DispatchThreadID \)/void DlssRrPrepareInputsMain( uint3 dispatchThreadID )/' \
         -e 's/(^|[^A-Za-z0-9_.])([0-9]+[eE][-+]?[0-9]+)([^0-9A-Za-z_.]|$)/\1\2f\3/g'
}
echo; echo "#line 94 \"$PP\""; filter "$PP" | sed -n '94,160p' | pass
echo; echo '#define DENOISER_DLSS_RR 1'
echo "#line 175 \"$PP\""; filter "$PP" | sed -n '175,440p' | pass
echo '#endif'
echo; echo '#define DLSS_RR_KAT_DRIVER 1'
echo '#include "ref_kat_dlss_rr_main.cpp"'
