"""GPU: cost of stochastic texture filtering (rtxpt_b200_set_texture_filtering) on bench.py's workload (city block 1920x1080, reference mode): frame time of a plain context
and per-kernel times (k_shade and the rest) from a second context with RTXPT_CFG_TIME_KERNELS (CUDA events around every kernel, kernels back to back), with STF off and with
the Linear, Cubic and Gaussian (sigma 0.3) filters.  Rounds rotate the order of the four settings.  The card's name, power limit and maximum SM clock are read at the start, the
SM clock and the throttle reasons after every timed block.  Prints one JSON line and writes it to --out/stf.json.

    python scripts/bench_stf.py --out DIR [--frames 6] [--rounds 3]
"""
import argparse, json, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]
from bench_approximate_mis import smi, clock_now, reference_frames  # noqa: E402

SETTINGS = {"off": None, "linear": 1, "cubic": 2, "gaussian": 3}


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--frames", type=int, default=6); ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from bench import build_workload, SPP
    from rtxpt_b200 import lib, structs as S
    name, power, max_sm = smi("name,power.limit,clocks.max.sm")
    res = {"gpu": {"device": name, "power_limit": power, "max_sm_clock": max_sm}, "reference": {}}
    scene, consts = build_workload()
    c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene)
    ct = lib.Context(max_sub_samples_per_launch=SPP, flags=S.CFG_TIME_KERNELS); ct.upload_scene(scene)
    keys = list(SETTINGS)
    runs = {k: {"ms": [], "kernels": [], "clocks": []} for k in keys}
    for rnd in range(args.rounds):
        for k in keys[rnd % 4:] + keys[:rnd % 4]:
            for x in (c, ct): x.set_texture_filtering(SETTINGS[k] is not None, SETTINGS[k] or 0, 0, 0.3)
            t, _ = reference_frames(c, consts, SPP, args.frames); runs[k]["ms"].append(t["msTotal"]); runs[k]["clocks"].append(clock_now())
            kt, _ = reference_frames(ct, consts, SPP, max(2, args.frames // 2)); runs[k]["kernels"].append(kt)
    for k in keys:
        r = runs[k]
        res["reference"][k] = {"ms_per_frame": statistics.median(r["ms"]), "ms_per_frame_runs": r["ms"],
                               "kernel_ms_back_to_back": {m: statistics.median(x[m] for x in r["kernels"]) for m in r["kernels"][0]},
                               "clocks_after_runs": r["clocks"]}
    c.close(); ct.close()
    res["workload"] = "bench.py: city block 1920x1080, %d spp, 6 bounces, NEE 5 candidates, reference mode" % SPP
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "stf.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
