#!/usr/bin/env bash
# ORACLE/_ref — TEST INFRASTRUCTURE.  Writes ONE C++ translation unit to stdout for ref_kat_stf_main.cpp: ref_hlsl_shim.h, the driver's stand-ins, then the UNMODIFIED RTXTF headers
# (External/Rtxtf: STFDefinitions.h, STFMacros.hlsli, STFSamplerStateImpl.hlsli, STFSamplerState.hlsli) read from where they lie under $REF through the spelling filter of
# ref_hlsl_tu.sh (taken from that script, so both streams rewrite the same spellings), then the driver.  Nothing of the reference is written to disk.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
eval "$(sed -n '/^filter() {/,/^}/p' "$HERE/ref_hlsl_tu.sh")"
STF=$REF/External/Rtxtf
echo '#include "ref_hlsl_shim.h"'
echo '#define STF_KAT_STANDINS 1'
echo '#include "ref_kat_stf_main.cpp"'
echo '#undef STF_KAT_STANDINS'
for f in STFDefinitions.h STFMacros.hlsli STFSamplerStateImpl.hlsli STFSamplerState.hlsli; do
  # HLSL converts int2 to float2 implicitly where the shim's vectors want it spelled: the coordinates handed to _GetFilterPDF
  echo; echo "#line 1 \"$STF/$f\""; filter "$STF/$f" | sed -E 's/_GetFilterPDF\(texelCoord, (coord[A-Za-z]+)\)/_GetFilterPDF(texelCoord, float2(\1))/g'
done
echo; echo '#include "ref_kat_stf_main.cpp"'
