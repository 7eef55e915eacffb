"""GPU: cost of the two light-vs-BSDF MIS kinds (RtxptPathTracerConstants::useApproximateMIS 0 = full, 1 = approximate) on two workloads:
  reference  bench.py's workload (city block 1920x1080, 4 spp, 6 bounces, reference mode): frame time of a plain context, and per-kernel times (k_trace_closest, k_trace_shadow,
             k_shade, other) from a second context with RTXPT_CFG_TIME_KERNELS (CUDA events around every kernel, kernels back to back)
  config3    BASELINE config 3's path tracing (city with delta surfaces 1920x1080, NEE-AT with temporal feedback, realtime mode, 4 FILL sub-samples): update_begin on the host clock
             and the path_trace_realtime call (BUILD + UpdateEnd + 4 x FILL) on CUDA events, after 16 warm-up frames; the ReBLUR denoiser and the tone mapper do not depend on the
             MIS kind and are left out
Rounds alternate the order of the two kinds.  The card's name, power limit and maximum SM clock are read at the start, the SM clock and the throttle reasons right after every
timed block.  Prints one JSON line and writes it to --out/approximate_mis.json.

    python scripts/bench_approximate_mis.py --out DIR [--frames 6] [--rounds 3]
"""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def smi(fields):
    q = subprocess.run(["nvidia-smi", "--query-gpu=" + fields, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return [x.strip() for x in q.split(",")]


def clock_now():
    out = {"sm_clock": smi("clocks.sm")[0]}
    try: out["throttle_reasons"] = smi("clocks_throttle_reasons.active")[0]
    except subprocess.CalledProcessError: out["throttle_reasons"] = "not reported"
    return out


def reference_frames(c, consts, spp, n):
    keys = ("msTotal", "msTraceClosest", "msTraceShadow", "msShade", "msOther")
    t = {k: [] for k in keys}
    for i in range(n + 1):
        consts.sampleBaseIndex = i * spp; c.set_constants(consts); c.path_trace(0, spp, True); c.synchronize()
        st = c.stats()
        if i:
            for k in keys: t[k].append(getattr(st, k))
    return {k: statistics.median(v) for k, v in t.items()}, st


def config3_frames(c, consts, spp, warm, n):
    ub, tr = [], []
    for f in range(warm + n):
        consts.sampleBaseIndex = f * spp; c.set_constants(consts)
        c.synchronize(); t0 = time.perf_counter(); c.neeat_update_begin(); c.synchronize(); t1 = time.perf_counter()
        c.path_trace_realtime(False); c.synchronize()
        if f >= warm: ub.append((t1 - t0) * 1e3); tr.append(float(c.stats().msTotal))
    return {"update_begin_ms": statistics.median(ub), "trace_ms": statistics.median(tr), "trace_ms_min": min(tr), "trace_ms_max": max(tr)}


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--frames", type=int, default=6); ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    from bench import build_workload, SPP
    from rtxpt_b200 import lib, scenes, scene_builder as sb, structs as S
    name, power, max_sm = smi("name,power.limit,clocks.max.sm")
    res = {"gpu": {"device": name, "power_limit": power, "max_sm_clock": max_sm}, "reference": {}, "config3": {}}
    # reference mode: the bench workload
    scene, consts = build_workload()
    c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene)
    ct = lib.Context(max_sub_samples_per_launch=SPP, flags=S.CFG_TIME_KERNELS); ct.upload_scene(scene)
    runs = {m: {"ms": [], "kernels": [], "clocks": []} for m in (0, 1)}; rays = {}
    for rnd in range(args.rounds):
        for m in ((0, 1) if rnd % 2 == 0 else (1, 0)):
            consts.useApproximateMIS = m
            t, st = reference_frames(c, consts, SPP, args.frames); runs[m]["ms"].append(t["msTotal"]); runs[m]["clocks"].append(clock_now())
            kt, _ = reference_frames(ct, consts, SPP, max(2, args.frames // 2)); runs[m]["kernels"].append(kt)
            rays[m] = (int(st.scatterRays), int(st.shadowRays))
    for m in (0, 1):
        r = runs[m]; ms = statistics.median(r["ms"])
        res["reference"][str(m)] = {"ms_per_frame": ms, "ms_per_frame_runs": r["ms"], "mrays_per_s": sum(rays[m]) / (ms * 1e-3) / 1e6, "scatter_shadow_rays": rays[m],
                                    "kernel_ms_back_to_back": {k: statistics.median(x[k] for x in r["kernels"]) for k in r["kernels"][0]},
                                    "kernel_ms_runs": r["kernels"], "clocks_after_runs": r["clocks"]}
    c.close(); ct.close(); del scene
    # config 3: realtime mode with NEE-AT feedback
    W, H, SPP3 = 1920, 1080, 4
    scene, cam = scenes.city_block(target_triangles=2_800_000, width=W, height=H, delta_surfaces=True)
    k = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2); k.NEEATFeedback = 1
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=SPP3)
    runs3 = {m: {"t": [], "clocks": []} for m in (0, 1)}
    ctxs = {}
    for m in (0, 1):
        k.useApproximateMIS = m
        x = lib.Context(max_sub_samples_per_launch=1); x.upload_scene(scene); x.set_constants(k); x.set_view(sb.world_to_clip(cam)); x.set_realtime(rt); ctxs[m] = x
    for rnd in range(args.rounds):
        for m in ((0, 1) if rnd % 2 == 0 else (1, 0)):
            k.useApproximateMIS = m
            runs3[m]["t"].append(config3_frames(ctxs[m], k, SPP3, 16 if rnd < 2 else 4, 10)); runs3[m]["clocks"].append(clock_now())
    for m in (0, 1):
        res["config3"][str(m)] = {"trace_ms": statistics.median(t["trace_ms"] for t in runs3[m]["t"]), "update_begin_ms": statistics.median(t["update_begin_ms"] for t in runs3[m]["t"]),
                                  "runs": runs3[m]["t"], "clocks_after_runs": runs3[m]["clocks"]}
        ctxs[m].close()
    res["workloads"] = {"reference": "bench.py: city block 1920x1080, %d spp, 6 bounces, NEE 5 candidates" % SPP,
                        "config3": "city block with delta surfaces 1920x1080, NEE-AT with feedback, realtime BUILD + UpdateEnd + 4 FILL sub-samples (each context keeps its own NEE-AT history)"}
    line = json.dumps(res)
    print(line)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "approximate_mis.json"), "w") as f: f.write(line + "\n")


if __name__ == "__main__":
    main()
