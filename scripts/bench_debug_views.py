"""GPU: cost of a first-hit debug view (rtxpt_b200_set_debug_view) on bench.py's workload (city block 1920x1080, reference mode): frame time with the view off and with
FirstHit_ShadingNormal, alternating the two in every round.  The card's name, power limit and maximum SM clock are read at the start, the SM clock after every timed block.
Prints one JSON line and writes it to --out/debug_views.json.

    python scripts/bench_debug_views.py --out DIR [--frames 6] [--rounds 3]
"""
import argparse, json, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
from bench_approximate_mis import smi, clock_now, reference_frames  # noqa: E402


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--frames", type=int, default=6); ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from bench import build_workload, SPP
    from rtxpt_b200 import lib, structs as S
    name, power, max_sm = smi("name,power.limit,clocks.max.sm")
    res = {"gpu": {"device": name, "power_limit": power, "max_sm_clock": max_sm}, "reference": {}}
    scene, consts = build_workload()
    c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene)
    settings = {"off": S.DEBUG_VIEW["Disabled"], "FirstHit_ShadingNormal": S.DEBUG_VIEW["FirstHit_ShadingNormal"]}
    runs = {k: {"ms": [], "clocks": []} for k in settings}
    keys = list(settings)
    for rnd in range(args.rounds):
        for k in keys[rnd % 2:] + keys[:rnd % 2]:
            c.set_debug_view(settings[k])
            t, _ = reference_frames(c, consts, SPP, args.frames); runs[k]["ms"].append(t["msTotal"]); runs[k]["clocks"].append(clock_now())
    for k in keys:
        res["reference"][k] = {"ms_per_frame": statistics.median(runs[k]["ms"]), "ms_per_frame_runs": runs[k]["ms"], "clocks_after_runs": runs[k]["clocks"]}
    c.close()
    res["workload"] = "bench.py: city block 1920x1080, %d spp, 6 bounces, NEE 5 candidates, reference mode" % SPP
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "debug_views.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
