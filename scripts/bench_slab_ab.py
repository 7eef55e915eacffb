"""GPU: A/B of builds of the product library on the bench workload - the measurement behind a change to the traversal's node step (traverse.cuh: nodeHitMask).

Runs `bench.py --steps 30 --warmup 3 --no-cpu-baseline` once per library and round with RTXPT_LIB pointing at that library (rtxpt_b200/lib.py), the libraries alternating inside
every round so that drift of the card hits all of them alike.  The first library is the baseline.  Round 0 also runs the realtime section (config 3) and dumps the accumulated
frame; the later rounds pass --no-realtime.  Reports, per library: every round's ms/frame, the serialised kernel times, the card's clocks during the timed window, config 3's
frame time, the range of node visits per ray (the counted steps depend on when a lane learns of a nearer hit, so they differ in the fifth digit from run to run of one
library); and against the baseline: whether the accumulated frame is bit-identical, whether the ray counts are equal, whether every run beats every baseline run, and the
difference of the medians.  The card's name and power limit are read at the start.  Prints the report and writes --out/slab_ab.json.

    make -C rtxpt_b200/csrc variant NAME=i2f1 EXTRA=-DPT_I2F_AXES=1
    python scripts/bench_slab_ab.py --out DIR old=/path/to/parent/librtxpt_b200.so new=rtxpt_b200/csrc/_build/librtxpt_b200.so i2f1=rtxpt_b200/csrc/_build/librtxpt_b200_var_i2f1.so
"""
import argparse, json, os, statistics, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"device": name, "power_limit": power}


def bench(lib_path, dump_dir, realtime, steps, warmup):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline"]
    if not realtime: cmd.append("--no-realtime")
    if dump_dir: cmd += ["--dump-outputs", dump_dir]
    r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, RTXPT_LIB=os.path.abspath(lib_path)))
    if r.returncode != 0: raise SystemExit("bench.py failed with %s:\n%s" % (lib_path, r.stderr[-2000:]))
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30); ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("libs", nargs="+", help="name=path of a library, the baseline first")
    args = ap.parse_args()
    libs = [x.split("=", 1) for x in args.libs]
    for name, path in libs:
        if not os.path.exists(path): raise SystemExit("%s: %s is missing" % (name, path))
    os.makedirs(args.out, exist_ok=True)
    report = {"gpu": gpu_info(), "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "runs": {name: [] for name, _ in libs}}
    for rnd in range(args.rounds):
        for name, path in (libs if rnd % 2 == 0 else libs[::-1]):
            line = bench(path, os.path.join(args.out, "dump_" + name) if rnd == 0 else None, rnd == 0, args.steps, args.warmup)
            k = line["roofline"]["kernel_ms_per_frame"]
            run = {"ms_per_frame": line["ms_per_step"], "mrays_s": line["value"], "trace_closest": k["trace_closest"], "trace_shadow": k["trace_shadow"], "shade": k["shade"],
                   "clocks": line["clocks"], "nodes_per_ray": line["roofline"]["nodes_per_ray"], "tris_per_ray": line["roofline"]["tris_per_ray"],
                   "scatter_rays": line["scatter_rays"], "shadow_rays": line["shadow_rays"], "rays_per_iteration": line["rays_per_iteration"]}
            if rnd == 0:
                c3 = line.get("config3") or {}
                run["config3"] = {k3: v for k3, v in c3.items() if isinstance(v, (int, float))} if isinstance(c3, dict) else c3
            report["runs"][name].append(run)
            print("round %d %-8s %.3f ms/frame  closest %.2f shadow %.2f shade %.2f  %s" % (rnd, name, run["ms_per_frame"], run["trace_closest"], run["trace_shadow"], run["shade"], json.dumps(run["clocks"])), flush=True)
    base = libs[0][0]; b = report["runs"][base]
    frame0 = np.load(os.path.join(args.out, "dump_" + base, "accumulated.npy"))
    report["against_" + base] = {}
    for name, _ in libs[1:]:
        r = report["runs"][name]
        same_counts = all(x[key] == b[0][key] for x in r for key in ("scatter_rays", "shadow_rays", "rays_per_iteration"))
        report["against_" + base][name] = {
            "accumulated_bit_identical": bool(np.array_equal(frame0.view(np.uint32), np.load(os.path.join(args.out, "dump_" + name, "accumulated.npy")).view(np.uint32))),
            "ray_counts_equal": same_counts,
            "every_run_beats_every_baseline_run": max(x["ms_per_frame"] for x in r) < min(x["ms_per_frame"] for x in b),
            "median_ms_per_frame": [statistics.median(x["ms_per_frame"] for x in b), statistics.median(x["ms_per_frame"] for x in r)],
            "median_gain_ms": statistics.median(x["ms_per_frame"] for x in b) - statistics.median(x["ms_per_frame"] for x in r)}
    with open(os.path.join(args.out, "slab_ab.json"), "w") as f: json.dump(report, f, indent=1)
    print(json.dumps({"gpu": report["gpu"], "against_" + base: report["against_" + base],
                      "ms_per_frame": {n: [round(x["ms_per_frame"], 3) for x in v] for n, v in report["runs"].items()},
                      "nodes_per_ray": {n: [min(x["nodes_per_ray"] for x in v), max(x["nodes_per_ray"] for x in v)] for n, v in report["runs"].items()},
                      "config3": {n: v[0].get("config3") for n, v in report["runs"].items()}}))


if __name__ == "__main__":
    main()
