"""GPU: cost of rtxpt_b200_update_env_map on the bench workload (bench.py: city block, 1920x1080, 4 spp, 6 bounces) against today's route, bake_env_map + upload_scene.

A seeded 4096x2048 equirectangular source and a sun that moves on every call, at cubeDim 1024 and 2048.  Reports, per cube size: the median host-clock time of the synchronous
update call and the median of its CUDA-event split (bake, importance map, copy into the cube array, read-back + host light bake + upload), the time of bake_env_map +
upload_scene of the same cube, and the frame time after an update and after a fresh upload of the same cube (rounds alternate the two).  Prints one JSON line and writes it
to --out/env_update.json.

    python scripts/bench_env_update.py --out DIR [--updates 10] [--frames 4] [--rounds 2]
"""
import argparse, json, os, statistics, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import numpy as np


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in q.split(",")]
    return {"device": name, "power_limit": power}


def sun(i):
    t = 0.05 * i
    d = np.float32([0.6 * np.cos(t), -0.5 - 0.3 * np.sin(t), 0.6 * np.sin(t)]); d /= np.linalg.norm(d)
    return [((1.0, 0.93, 0.82), 60.0, tuple(float(x) for x in d), 0.0093)]


def set_cube(scene, mips):
    """Points the scene description's environment cube at `mips` (kept alive on the scene object)."""
    d = scene.desc.envCube; d.faceSize, d.mipLevels = mips[0].shape[1], len(mips)
    scene._bench_cube = [np.ascontiguousarray(m) for m in mips]
    for m, arr in enumerate(scene._bench_cube):
        for f in range(6): d.faces[f][m] = arr[f].ctypes.data


def frame_ms(c, consts, spp, frames):
    t = []
    for i in range(frames + 1):
        consts.sampleBaseIndex = i * spp; c.set_constants(consts); c.path_trace(0, spp, True); c.synchronize()
        if i: t.append(c.stats().msTotal)
    return statistics.median(t)


def main():
    ap = argparse.ArgumentParser(); ap.add_argument("--out", required=True); ap.add_argument("--updates", type=int, default=10); ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2); ap.add_argument("--dims", default="1024,2048")
    args = ap.parse_args()
    from bench import build_workload, SPP
    from rtxpt_b200 import lib
    info = gpu_info()
    scene, consts = build_workload()
    source = np.random.default_rng(2048).gamma(2.0, 0.5, (2048, 4096, 4)).astype(np.float32)
    res = {}
    for dim in [int(x) for x in args.dims.split(",")]:
        r = {}
        c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene); c.set_constants(consts)
        c.update_env_map(dim, source, lights=sun(0))                                      # first call: scratch, cube array and kept source allocated
        wall, split = [], []
        for i in range(1, args.updates + 1):
            t0 = time.perf_counter(); c.update_env_map(dim, kept_source=(1, 4096, 2048), lights=sun(i)); wall.append(time.perf_counter() - t0)
            split.append(c.last_env_update_ms())
        r["update_ms_call_median"] = 1e3 * statistics.median(wall)
        r["update_ms_events_median"] = {k: statistics.median(s[k] for s in split) for k in split[0]}
        t0 = time.perf_counter(); c.update_env_map(dim, source, lights=sun(0)); r["update_with_new_source_ms"] = 1e3 * (time.perf_counter() - t0)
        mips = c.bake_env_map(dim, source, lights=sun(args.updates)); c.close()
        # today's route: bake to host memory, then a full upload of the scene with that cube
        route = []
        for k in range(2):
            c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene); c.set_constants(consts)
            t0 = time.perf_counter(); m = c.bake_env_map(dim, source, lights=sun(k)); set_cube(scene, m); c.upload_scene(scene); c.set_constants(consts); route.append(time.perf_counter() - t0)
            c.close()
        r["bake_and_upload_ms_median"] = 1e3 * statistics.median(route)
        # frames: after an update and after a fresh upload of the same cube
        set_cube(scene, mips)
        fr = {"after_update": [], "after_upload": []}
        for rnd in range(args.rounds):
            for kind in (("after_update", "after_upload") if rnd % 2 == 0 else ("after_upload", "after_update")):
                c = lib.Context(max_sub_samples_per_launch=SPP); c.upload_scene(scene); c.set_constants(consts)
                if kind == "after_update": c.update_env_map(dim, source, lights=sun(args.updates))
                fr[kind].append(frame_ms(c, consts, SPP, args.frames)); c.close()
        r["frame_ms"] = fr
        res[str(dim)] = r
    out = {**info, "cube_dims": res, "source": "4096x2048 RGBA32F equirectangular, seeded; one directional light moving on every call", "updates": args.updates,
           "timing": "update: host clock around the synchronous call (median of warm calls from the kept source), split by the call's CUDA events (last_env_update_ms); "
                     "bake_and_upload: host clock around bake_env_map + upload_scene + set_constants; frame: stats().msTotal, median of warm frames of 4 spp"}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "env_update.json"), "w") as f: json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
