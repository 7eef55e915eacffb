"""Times realtime mode (SURVEY §8 row a17: stable-plane BUILD pass + FILL pass + no-denoiser merge) on bench.py's city workload and prints ONE JSON object.
Run by bench.py in a child process after the headline measurement (a failure here must not cost the headline line), or by hand on a GPU box:
    python scripts/bench_realtime.py [--frames 10] [--sub-samples 1]
Clear glass (roughness below the delta threshold) is opted into the path-space decomposition the way a .material.json with PSDExclude = false does, so the BUILD pass
has real forks to explore; everything else keeps RTXPT's default (excluded)."""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def measured_peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        with open(p) as f: return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    except Exception:  # noqa: BLE001
        return 3350.0, "fallback (H100 SXM data sheet: 3.35 TB/s HBM3)"


def config3(args, lib, scenes, sb, S):
    W, H, SPP, WARM = args.width, args.height, 4, 32
    scene, cam = scenes.city_block(target_triangles=args.triangles, width=W, height=H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    consts.NEEATFeedback = 1
    ctx = lib.Context(max_sub_samples_per_launch=1)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=SPP); ctx.set_realtime(rt)
    k = sb.make_denoiser_constants(cam); tm = S.make_tone_mapping_params(op=5, auto_exposure=True)
    ev = {key: [] for key in ("update_begin_ms", "trace_ms", "denoise_ms", "frame_ms")}
    for f in range(WARM + args.frames):
        consts.sampleBaseIndex = f * SPP; ctx.set_constants(consts)
        ctx.synchronize(); t0 = time.perf_counter()
        ctx.neeat_update_begin(); ctx.synchronize(); t1 = time.perf_counter()
        ctx.path_trace_realtime(False); ctx.synchronize(); trace = float(ctx.stats().msTotal)
        ctx.denoise_spec_hit_t()
        ctx.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=f, frame_time_ms=16.0)); dn = ctx.last_denoise_ms()
        ctx.tone_map(tm); ctx.synchronize(); t2 = time.perf_counter()
        if f >= WARM:
            ev["update_begin_ms"].append((t1 - t0) * 1e3); ev["trace_ms"].append(trace); ev["denoise_ms"].append(dn); ev["frame_ms"].append((t2 - t0) * 1e3)
    st = ctx.stats(); r = ctx.readback_realtime(); hd = r["header"]
    img = ctx.readback_output_color()[..., :3].astype(np.float32); ctl = ctx.neeat_raw(8, np.uint32, 8)
    planes = [float((hd[p] != 0xFFFFFFFF).mean()) for p in range(3)]
    med = {key: float(np.median(v)) for key, v in ev.items()}
    peak, peak_src = measured_peak_gbs()
    px = W * H; bytes_per_plane = 190 * px                      # SURVEY §8(d): inputs 33 + permanent pool r/w 2 x 42 + transient r/w 2 x 28 + outputs 16 B per pixel, taps assumed cached
    rays = int(st.scatterRays + st.shadowRays)                  # the last FILL sub-sample's counters
    out = dict(med)
    out.update({"image": [W, H], "spp": SPP, "warmup_frames": WARM, "frames": args.frames, "emissive_triangle_lights": int(st.lightCount) - 5368, "planes_denoised": 3,
                "pixels_with_plane": planes, "pixels_with_feedback": float(ctl[7]) / float(px), "sampling_proxies": int(ctl[4]), "finite": bool(np.isfinite(img).all()), "mean_radiance": float(img.mean()),
                "kernel_launches_trace": int(st.kernelLaunches), "fill_rays_last_sub_sample": rays,
                "reblur_roofline": {"bound": "hbm (compulsory bytes; the passes are ALU-heavy)", "algorithmic_bytes_per_plane": int(bytes_per_plane), "planes": 3,
                                    "achieved": 3 * bytes_per_plane / (med["denoise_ms"] * 1e-3) / 1e9, "peak": peak, "unit": "GB/s", "frac": 3 * bytes_per_plane / (med["denoise_ms"] * 1e-3) / 1e9 / peak,
                                    "peak_source": peak_src, "note": "denoise_ms covers, per plane, prepare inputs + 8 ReBLUR passes + final merge; every plane is charged the full frame although planes 1-2 cover only pixels_with_plane[1..2] of it"},
                "timing": "update_begin_ms, frame_ms: host clock between synchronizes; trace_ms (BUILD + UpdateEnd + 4 x FILL), denoise_ms: CUDA events on the context stream; medians over the timed frames"})
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=10); ap.add_argument("--warmup", type=int, default=3); ap.add_argument("--sub-samples", type=int, default=1)
    ap.add_argument("--width", type=int, default=1920); ap.add_argument("--height", type=int, default=1080); ap.add_argument("--triangles", type=int, default=2_800_000)
    args = ap.parse_args()
    real_stdout = os.dup(1); os.dup2(2, 1)
    from rtxpt_b200 import lib, scenes, scene_builder as sb, structs as S
    W, H = args.width, args.height
    scene, cam = scenes.city_block(target_triangles=args.triangles, width=W, height=H)
    opted = 0
    for i in range(scene.desc.materialCount):
        m = scene.desc.materials[i]
        if m.TransmissionFactor > 0 and m.Roughness * m.Roughness < 0.0064:
            m.Flags = (m.Flags & ~S.MATFLAG_PSDExclude & ~0x0F000000) | (1 << 24); opted += 1          # PSDExclude off, dominant delta lobe = transmission
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    ctx = lib.Context(max_sub_samples_per_launch=1)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=args.sub_samples)
    ctx.set_realtime(rt)
    ms = []
    for f in range(args.warmup + args.frames):
        consts.sampleBaseIndex = f * args.sub_samples; ctx.set_constants(consts)
        ctx.path_trace_realtime(True); ctx.synchronize()
        st = ctx.stats()
        if f >= args.warmup: ms.append(float(st.msTotal))
    r = ctx.readback_realtime()
    hd = r["header"]
    out = {"ms_per_frame": float(np.median(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)), "frames": args.frames, "warmup": args.warmup,
           "image": [W, H], "sub_samples": args.sub_samples, "active_planes": 3, "max_vertex_depth": int(rt.maxStablePlaneVertexDepth), "kernel_launches_per_frame": int(st.kernelLaunches),
           "materials_opted_into_decomposition": opted, "fill_pass_scatter_rays": int(st.scatterRays), "fill_pass_shadow_rays": int(st.shadowRays),
           "pixels_with_plane": [float((hd[p] != 0xFFFFFFFF).mean()) for p in range(3)], "pixels_with_non_primary_dominant_plane": float(((hd[3] & 3) != 0).mean()),
           "mean_radiance": float(r["merged"].mean()), "timing": "CUDA events around the whole rtxpt_b200_path_trace_realtime call (BUILD + FILL x sub_samples + merge), median over frames",
           "workload": "bench.py city workload, clear glass opted into path-space decomposition"}
    # ---- BASELINE configs[2]: "1080p, 4 spp, NEE-AT + 10k emissive triangles + ReBLUR denoise" --------------------------------------------------------------------------------
    # One frame = what Sample::Render does in realtime mode: LightsBaker::UpdateBegin -> BUILD -> LightsBaker::UpdateEnd -> 4 x FILL (NEE with local + global candidates, feedback)
    # -> DenoiseSpecHitT -> per plane { prepare inputs, ReBLUR (8 passes), final merge } -> tone map.  32 warm-up frames prime the NEE-AT caches (Sample.cpp:1423) and the ReBLUR
    # history.  Scene: the city workload with delta surfaces (glazed shop fronts, wet street) so that stable planes 1 and 2 are populated; >= 10 k emissive triangles (street lamps).
    try:
        out["config3"] = config3(args, lib, scenes, sb, S)
    except Exception as e:  # noqa: BLE001
        out["config3"] = {"error": repr(e)[:400]}
    # the callers either side of the path (§8f rows 3-4), first GPU executions as well: tone mapping, environment bake, BVH refit (last: a wrong refit would spoil what follows)
    try:
        tm = S.make_tone_mapping_params(op=5, auto_exposure=True); ctx.tone_map(tm); ctx.synchronize()
        t0 = time.perf_counter()
        for _ in range(10): ctx.tone_map(tm)
        ctx.synchronize(); tone_ms = (time.perf_counter() - t0) * 100.0
        ldr = ctx.readback_ldr()
        eq = np.random.default_rng(1).gamma(2.0, 0.5, (256, 512, 4)).astype(np.float32)
        t0 = time.perf_counter(); mips = ctx.bake_env_map(512, eq, lights=[((1.0, 0.9, 0.8), 10.0, (0.3, -0.8, 0.52), 0.05)]); bake_ms = (time.perf_counter() - t0) * 1e3
        n_inst = scene.desc.instanceCount
        xf = np.stack([np.array(scene.desc.instances[i].transform[:], np.float32).reshape(3, 4) for i in range(n_inst)])
        ctx.update_instance_transforms(xf); ctx.synchronize()
        t0 = time.perf_counter()
        for _ in range(5): ctx.update_instance_transforms(xf)
        ctx.synchronize(); refit_ms = (time.perf_counter() - t0) * 200.0
        consts.sampleBaseIndex = 0; ctx.set_constants(consts); ctx.path_trace_realtime(True); ctx.synchronize()
        after = float(ctx.readback_output_color()[..., :3].astype(np.float32).mean())
        out["callers"] = {"tone_map_ms_host_clock": tone_ms, "tone_map_avg_luminance": ctx.tone_map_average_luminance(), "ldr_mean": float(ldr[..., :3].mean()),
                          "env_bake_512_ms_host_clock_incl_copies": bake_ms, "env_bake_finite": bool(np.isfinite(mips[0]).all()),
                          "bvh_refit_ms_host_clock": refit_ms, "instances": int(n_inst), "bvh_intact_after_identity_refit": bool(abs(after - out["mean_radiance"]) < 0.25 * abs(out["mean_radiance"]) + 1e-6)}
    except Exception as e:  # noqa: BLE001
        out["callers"] = {"error": repr(e)[:300]}
    os.write(real_stdout, (json.dumps(out) + "\n").encode())         # before teardown: a device fault in the untested stage must not cost the line
    try: ctx.close()
    except Exception: pass  # noqa: BLE001
    return 0


if __name__ == "__main__":
    sys.exit(main())
