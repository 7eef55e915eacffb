"""Workload for the `ncu --set full` capture of the wavefront kernels (summarised under profiles/ by scripts/ncu_summary.py): bench.py's frame (city, 1920x1080, 4 spp, 6 bounces), 3 frames.
One frame = k_generate + 11 x (k_trace_closest, k_shade, k_trace_shadow) + k_commit_accumulate = 35 launches; the third frame is captured:
    ncu --set full --clock-control none --import-source on -k regex:"k_generate|k_trace_|k_shade|k_commit" -s 70 -c 35 -o gpurun_out/r2_full python scripts/profile_wavefront.py"""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench
from rtxpt_b200 import lib

scene, consts = bench.build_workload()
ctx = lib.Context(max_sub_samples_per_launch=bench.SPP)
ctx.upload_scene(scene); ctx.set_constants(consts)
for f in range(int(os.environ.get("FRAMES", "3"))):
    consts.sampleBaseIndex = f * bench.SPP; ctx.set_constants(consts)
    ctx.path_trace(0, bench.SPP, True); ctx.synchronize()
st = ctx.stats(); print("rays per frame", st.scatterRays + st.shadowRays, "launches", st.kernelLaunches, "ms", st.msTotal)
ctx.close()
