"""GPU: cost of NEEFullSamples (light samples per path vertex, each with its own shadow ray) on the bench workload (bench.py: city block, 1920x1080, 4 spp, 6 bounces).

For N = 1, 2, 4 (rounds alternate the order): the median frame time, rays per second (scatter + shadow), shadow rays per frame, sub-samples per launch, and from a second
context with per-kernel CUDA events (RTXPT_CFG_TIME_KERNELS, kernels back to back) the time of each kernel kind; msOther holds generate, commit and - for N > 1 - k_nee_resolve,
so its growth over N = 1 is the resolve.  The card's name and power limit are read at the start.  Prints one JSON line and writes it to --out/nee_full_samples.json.

    python scripts/bench_nee_full_samples.py --out DIR [--frames 6] [--rounds 2] [--full 1,2,4]
"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"device": name, "power_limit": power}


def frames(c, consts, spp, n):
    """n timed frames after one warm-up frame: medians of msTotal and of the kernel-kind times, and the last frame's ray counts"""
    keys = ("msTotal", "msTraceClosest", "msTraceShadow", "msShade", "msOther")
    t = {k: [] for k in keys}
    for i in range(n + 1):
        consts.sampleBaseIndex = i * spp; c.set_constants(consts); c.path_trace(0, spp, True); c.synchronize()
        st = c.stats()
        if i:
            for k in keys: t[k].append(getattr(st, k))
    return {k: statistics.median(v) for k, v in t.items()}, st


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--frames", type=int, default=6); ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--full", default="1,2,4")
    args = ap.parse_args()
    from bench import build_workload, SPP
    from rtxpt_b200 import lib, structs as S
    info = gpu_info()
    scene, consts = build_workload()
    fulls = [int(x) for x in args.full.split(",")]
    c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene)
    ct = lib.Context(max_sub_samples_per_launch=SPP, flags=S.CFG_TIME_KERNELS); ct.upload_scene(scene)
    runs = {n: {"ms": [], "kernels": []} for n in fulls}
    stats = {}
    for rnd in range(args.rounds):
        for n in (fulls if rnd % 2 == 0 else fulls[::-1]):
            consts.NEEFullSamples = n
            t, st = frames(c, consts, SPP, args.frames)
            runs[n]["ms"].append(t["msTotal"]); stats[n] = st
            kt, _ = frames(ct, consts, SPP, max(2, args.frames // 2))
            runs[n]["kernels"].append(kt)
    res = {"gpu": info, "workload": "bench.py: city block 1920x1080, %d spp, 6 bounces, NEE 5 candidates" % SPP, "by_full_samples": {}}
    for n in fulls:
        ms = statistics.median(runs[n]["ms"]); st = stats[n]
        k = {key: statistics.median(r[key] for r in runs[n]["kernels"]) for key in runs[n]["kernels"][0]}
        res["by_full_samples"][str(n)] = {
            "ms_per_frame": ms, "ms_per_frame_runs": runs[n]["ms"],
            "mrays_per_s": (st.scatterRays + st.shadowRays) / (ms * 1e-3) / 1e6,
            "scatter_rays_per_frame": int(st.scatterRays), "shadow_rays_per_frame": int(st.shadowRays),
            "sub_samples_per_launch": max(1, SPP // n) if n > 1 else SPP,
            "kernel_ms_back_to_back": k,
        }
    base = res["by_full_samples"][str(fulls[0])]["kernel_ms_back_to_back"]["msOther"]
    for n in fulls:
        r = res["by_full_samples"][str(n)]; r["resolve_ms_estimate"] = r["kernel_ms_back_to_back"]["msOther"] - base if n > 1 else 0.0
    c.close(); ct.close()
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "nee_full_samples.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
