"""GPU: cost and effect of rtxpt_b200_rebuild_bvh on the bench workload (bench.py: 2.86 M-triangle city, 1920x1080, 4 spp, 6 bounces).

Reports the host build at upload, the device rebuild (CUDA events from bvh_stats().buildSeconds and the host clock around the whole call, which includes its waits; median of
warm rebuilds), the device memory the first rebuild takes (scratch + the second tree), and for four trees - the host build, the rebuild of the static scene, a far-moved scene
refitted only and the same scene rebuilt - their SAH expectations, the traversal steps per ray (RTXPT_CFG_COUNT_TRAVERSAL_STEPS) and the kernel times of a frame
(RTXPT_CFG_TIME_KERNELS), in alternating rounds.  Prints one JSON line and writes it to --out/bvh_rebuild.json.

    python scripts/bench_bvh_rebuild.py --out DIR [--rebuilds 20] [--rounds 2]
"""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"device": name, "power_limit": power}


def stats_dict(st):
    return {k: getattr(st, k) for k in ("nodeCount", "leafCount", "maxDepth", "expectedNodeVisits", "expectedTriangleTests", "buildSeconds")}


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--rebuilds", type=int, default=20); ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    from bench import build_workload, SPP
    from rtxpt_b200 import lib, structs as S
    from test_gpu_refit import mixed_motion
    info = gpu_info()
    scene, consts = build_workload()
    n = scene.desc.instanceCount
    far = mixed_motion(scene, far=True, fixed=(n - 1,))                                               # the emissive lamps stay where their lights were baked
    static = np.stack([np.float32(scene.instances[i].transform[:]).reshape(3, 4) for i in range(n)])

    # rebuild cost
    c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene); host = c.bvh_stats()
    torch.cuda.synchronize(); free0 = torch.cuda.mem_get_info()[0]
    c.update_instance_transforms(far); c.rebuild_bvh(); torch.cuda.synchronize(); free1 = torch.cuda.mem_get_info()[0]
    ev, wall = [], []
    for _ in range(args.rebuilds):
        t0 = time.perf_counter(); c.rebuild_bvh(); wall.append(time.perf_counter() - t0); ev.append(c.bvh_stats().buildSeconds)
    c.close()

    trees = {
        "host": lambda c: None,
        "rebuilt_static": lambda c: c.rebuild_bvh(),
        "far_refit_only": lambda c: c.update_instance_transforms(far),
        "far_rebuilt": lambda c: (c.update_instance_transforms(far), c.rebuild_bvh()),
    }
    res = {k: {"frame_ms": [], "closest_ms": [], "shadow_ms": [], "shade_ms": []} for k in trees}
    for rnd in range(args.rounds):
        for name, prep in (trees.items() if rnd % 2 == 0 else reversed(list(trees.items()))):
            c = lib.Context(max_sub_samples_per_launch=SPP, flags=S.CFG_TIME_KERNELS); c.upload_scene(scene); c.update_instance_transforms(static); prep(c)
            for i in range(4):
                consts.sampleBaseIndex = i * SPP; c.set_constants(consts); c.path_trace(0, SPP, True)
            c.synchronize(); s = c.stats()
            r = res[name]; r["frame_ms"].append(s.msTotal); r["closest_ms"].append(s.msTraceClosest); r["shadow_ms"].append(s.msTraceShadow); r["shade_ms"].append(s.msShade)
            r["sah"] = stats_dict(c.bvh_stats()); c.close()
            if rnd == 0:
                c = lib.Context(max_sub_samples_per_launch=SPP, flags=S.CFG_COUNT_TRAVERSAL_STEPS); c.upload_scene(scene); c.update_instance_transforms(static); prep(c)
                consts.sampleBaseIndex = 0; c.set_constants(consts); c.path_trace(0, SPP, True); c.synchronize(); s = c.stats(); c.close()
                r["nodes_per_ray"] = s.traversalNodeVisits / max(1, s.scatterRays); r["tris_per_ray"] = s.traversalTriTests / max(1, s.scatterRays)
    out = {"triangles": host.triangleReferenceCount, "host_build_s": host.buildSeconds,
           "rebuild_ms_events_median": 1e3 * statistics.median(ev), "rebuild_ms_call_median": 1e3 * statistics.median(wall), "rebuilds": args.rebuilds,
           "first_rebuild_device_bytes": int(free0 - free1), "trees": res, **info,
           "timing": "rebuild: CUDA events around the device work of one call (bvh_stats().buildSeconds) and the host clock around the call; frame: RTXPT_CFG_TIME_KERNELS contexts, "
                     "4 frames of 4 spp each, rounds alternate the order of the trees"}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bvh_rebuild.json"), "w") as f: json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
