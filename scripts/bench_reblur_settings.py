"""GPU: ReBLUR time under the settings RTXPT's denoiser panel exposes (rtxpt_b200_set_reblur_settings) on BASELINE configs[2]'s frame (scripts/bench_realtime.py config3: city
block 1920x1080 with delta surfaces, 4 spp, NEE-AT feedback, three stable planes).  The frame is traced and denoised for --warmup frames, then held: each timed call is one
rtxpt_b200_denoise_realtime on it (per plane: prepare inputs, the ReBLUR passes the settings select, final merge), timed by rtxpt_b200_last_denoise_ms (CUDA events).  Variants:
RTXPT's default (5x5 reconstruction, pre-pass radii 15 / 40), 3x3 reconstruction, reconstruction off, pre-pass off (both radii 0); each round runs every variant, in an order that
rotates from round to round.  The card's name, power limit and maximum SM clock are read at the start, the SM clock after every timed block.  Prints one JSON line and writes it
to --out/reblur_settings.json.

    python scripts/bench_reblur_settings.py --out DIR [--calls 20] [--rounds 4] [--warmup 8]
"""
import argparse, json, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]
from bench_approximate_mis import smi, clock_now  # noqa: E402


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--calls", type=int, default=20); ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=8); ap.add_argument("--width", type=int, default=1920); ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--triangles", type=int, default=2_800_000)
    args = ap.parse_args()
    from rtxpt_b200 import lib, scenes, scene_builder as sb, structs as S
    name, power, max_sm = smi("name,power.limit,clocks.max.sm")
    W, H, SPP = args.width, args.height, 4
    scene, cam = scenes.city_block(target_triangles=args.triangles, width=W, height=H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    consts.NEEATFeedback = 1
    ctx = lib.Context(max_sub_samples_per_launch=1)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.set_view(sb.world_to_clip(cam))
    ctx.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=SPP))
    k = sb.make_denoiser_constants(cam)
    variants = {"5x5 (default)": S.ReblurSettings.default(),
                "3x3": S.ReblurSettings.default(hitDistanceReconstructionMode=S.REBLUR_HIT_DISTANCE_RECONSTRUCTION_AREA_3X3),
                "reconstruction off": S.ReblurSettings.default(hitDistanceReconstructionMode=S.REBLUR_HIT_DISTANCE_RECONSTRUCTION_OFF),
                "pre-pass off": S.ReblurSettings.default(diffusePrepassBlurRadius=0.0, specularPrepassBlurRadius=0.0)}
    for f in range(args.warmup):
        consts.sampleBaseIndex = f * SPP; ctx.set_constants(consts)
        ctx.neeat_update_begin(); ctx.path_trace_realtime(False); ctx.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=f, frame_time_ms=16.0)); ctx.synchronize()
    keys = list(variants); runs = {v: {"ms": [], "clocks": []} for v in keys}; frame = args.warmup
    for rnd in range(args.rounds):
        for v in keys[rnd % len(keys):] + keys[:rnd % len(keys)]:
            ctx.set_reblur_settings(variants[v])
            ctx.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=frame, frame_time_ms=16.0)); ctx.last_denoise_ms(); frame += 1      # untimed: the first call after a change
            for _ in range(args.calls):
                ctx.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=frame, frame_time_ms=16.0)); runs[v]["ms"].append(ctx.last_denoise_ms()); frame += 1
            runs[v]["clocks"].append(clock_now())
    out = {"gpu": {"device": name, "power_limit": power, "max_sm_clock": max_sm},
           "workload": "BASELINE configs[2] frame: city block %dx%d, %d triangles, delta surfaces, %d spp, NEE-AT feedback, 3 stable planes; the traced frame held after %d warm-up frames"
                       % (W, H, args.triangles, SPP, args.warmup),
           "timing": "rtxpt_b200_last_denoise_ms (CUDA events around rtxpt_b200_denoise_realtime: 3 x { prepare inputs, ReBLUR, final merge } + the spec hit distance guide filter); "
                     "%d calls per variant per round, %d rounds, order rotated per round" % (args.calls, args.rounds),
           "denoise_ms": {v: {"median": statistics.median(runs[v]["ms"]), "min": min(runs[v]["ms"]), "max": max(runs[v]["ms"]),
                              "round_medians": [statistics.median(runs[v]["ms"][r * args.calls:(r + 1) * args.calls]) for r in range(args.rounds)], "clocks_after_rounds": runs[v]["clocks"]}
                          for v in keys}}
    ctx.close()
    line = json.dumps(out)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "reblur_settings.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
