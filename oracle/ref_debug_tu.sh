#!/usr/bin/env bash
# ORACLE/_ref — TEST INFRASTRUCTURE.  Writes ONE C++ translation unit to stdout for ref_kat_debug_main.cpp: ref_hlsl_shim.h, the driver's stand-ins, then the debug-view colour
# functions of the UNMODIFIED reference read from where they lie under $REF through the spelling filter of ref_hlsl_tu.sh (taken from that script): Unpack_R11G11B10_FLOAT
# (Utils/Packing.hlsli:186-192), GradientHeatMap and ColorFromHash (Utils/Utils.hlsli:92-112), StablePlaneDebugVizColor and StablePlaneDebugVizFourWaySplitCoord
# (StablePlanes.hlsli:314-335, the shader-only half included), DbgShowNormalSRGB (PathTracerShared.h:144-147); then the driver.  Nothing of the reference is written to disk.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
eval "$(sed -n '/^filter() {/,/^}/p' "$HERE/ref_hlsl_tu.sh")"
PT=$REF/Rtxpt/Shaders/PathTracer
echo '#include "ref_hlsl_shim.h"'
echo '#define DEBUG_KAT_STANDINS 1'
echo '#include "ref_kat_debug_main.cpp"'
echo '#undef DEBUG_KAT_STANDINS'
for f in Utils/Packing.hlsli:186-192 Utils/Utils.hlsli:92-112 StablePlanes.hlsli:314-335 PathTracerShared.h:144-147; do
  range=${f#*:}; f=${f%%:*}
  echo; echo "#line ${range%-*} \"$PT/$f\""; filter "$PT/$f" | sed -n "${range%-*},${range#*-}p"
done
echo; echo '#include "ref_kat_debug_main.cpp"'
