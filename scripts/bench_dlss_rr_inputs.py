"""GPU: time of RTXPT's DLSS-RR input pass (rtxpt_b200_dlss_rr_prepare_inputs) on BASELINE configs[2]'s frame (scripts/bench_realtime.py config3: city block 1920x1080 with delta
surfaces, 4 spp, three stable planes).  The frame is traced and its specular hit distance filtered once, then held: each timed block is --calls back-to-back calls on the caller's
stream between two CUDA events (1000 calls: a window of the order of 0.1 s at the expected time per call).  Bandwidth: the pass moves about NOMINAL_BYTES per pixel
(header 16 B, three 80 B plane records, stable radiance 8 B, hit distance 4 B, motion vectors 8 B in; 28 B out), reported over the measured time against the H100 SXM
data-sheet HBM3 peak, next to the card's name and power limit read in the same run.  The nominal count reads all three plane records; pixels whose planes 1 and 2 hold no branch
read less, so on this frame the nominal rate can exceed the peak: it bounds the traffic from above, it is not a measured byte count.  Measured on an H100 80GB HBM3 at 700 W:
0.159 ms per call (median of 10 blocks, spread 0.1 %).  Prints one JSON line and writes it to --out/dlss_rr_inputs.json.

    python scripts/bench_dlss_rr_inputs.py --out DIR [--calls 1000] [--blocks 10]
"""
import argparse, json, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]
from bench_approximate_mis import smi, clock_now  # noqa: E402

NOMINAL_BYTES = 16 + 3 * 80 + 8 + 4 + 8 + 28
HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes / s


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--calls", type=int, default=1000); ap.add_argument("--blocks", type=int, default=10)
    ap.add_argument("--width", type=int, default=1920); ap.add_argument("--height", type=int, default=1080); ap.add_argument("--triangles", type=int, default=2_800_000)
    args = ap.parse_args()
    import torch
    from rtxpt_b200 import lib, scenes, scene_builder as sb
    name, power, max_sm = smi("name,power.limit,clocks.max.sm")
    W, H, SPP = args.width, args.height, 4
    scene, cam = scenes.city_block(target_triangles=args.triangles, width=W, height=H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    ctx = lib.Context(max_sub_samples_per_launch=1)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.set_view(sb.world_to_clip(cam))
    ctx.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=SPP))
    ctx.path_trace_realtime(False); ctx.denoise_spec_hit_t(); ctx.synchronize()
    stream = torch.cuda.Stream(); s = stream.cuda_stream                       # a stream of its own: a null handle would send the calls to the context's stream
    for _ in range(5): ctx.dlss_rr_prepare_inputs(stream=s)                     # warm-up: allocation of the targets, module load
    stream.synchronize()
    per_call, clocks = [], []
    for _ in range(args.blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(args.calls): ctx.dlss_rr_prepare_inputs(stream=s)
        b.record(stream); b.synchronize()
        per_call.append(a.elapsed_time(b) / args.calls); clocks.append(clock_now())
    ms = statistics.median(per_call)
    gbs = NOMINAL_BYTES * W * H / (ms * 1e-3)
    out = {"gpu": {"device": name, "power_limit": power, "max_sm_clock": max_sm, "sm_clock_after_blocks": clocks},
           "workload": "BASELINE configs[2] frame: city block %dx%d, %d triangles, delta surfaces, %d spp, 3 stable planes; one traced frame held" % (W, H, args.triangles, SPP),
           "timing": "CUDA events around %d back-to-back rtxpt_b200_dlss_rr_prepare_inputs calls, %d blocks; median per call" % (args.calls, args.blocks),
           "ms": {"median": ms, "min": min(per_call), "max": max(per_call)},
           "nominal_bytes_per_pixel": NOMINAL_BYTES, "achieved_GBps": gbs / 1e9, "share_of_hbm_peak": gbs / HBM_PEAK}
    ctx.close()
    line = json.dumps(out)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "dlss_rr_inputs.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
