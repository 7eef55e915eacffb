"""GPU: realtime mode (SURVEY §8 row a17) - stable-plane BUILD / FILL passes and the no-denoiser merge of the CUDA path against the oracle, through
the C ABI (rtxpt_b200_set_realtime / rtxpt_b200_path_trace_realtime).  Integer state (branch IDs, dominant plane, vertex indices) must be identical;
packed fp16 / float fields are the oracle's on nearly every pixel in the strict (IEEE) build and within the stated tolerances in the default build
(libdevice vs glibc transcendentals, FMA contraction)."""
import numpy as np
import pytest

# Strict build: bit-identical to the oracle in every header word, plane field and guide; default build: identical in the decomposition except where a ray
# meets the glass box's bottom face and the floor at the same distance.  Fast-build tolerances marked "measured" come from GPU runs of these tests.
unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)

INVALID = 0xFFFFFFFF


def _halves(words):
    hi = (words >> 16).astype(np.uint16).view(np.float16).astype(np.float32); lo = (words & 0xFFFF).astype(np.uint16).view(np.float16).astype(np.float32)
    return hi, lo


def _setup(product, oracle, strict, W=96, H=96, bounces=8):
    from rtxpt_b200 import scene_builder as sb, scenes
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=bounces, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    return c, o, cam, consts


def _run_pair(product, oracle, strict, sub_samples=2):
    from rtxpt_b200 import scene_builder as sb
    W = H = 96
    c, o, cam, consts = _setup(product, oracle, strict, W, H)
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=sub_samples)
    c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    c.path_trace_realtime(True); c.synchronize(); g2 = c.readback_realtime()
    r = o.render_realtime(rt)
    c.close(); o.close()
    return g, g2, r, W, H


@pytest.mark.gpu
def test_realtime_strict_build_is_the_oracle(product, oracle):
    """IEEE build: the BUILD pass (branch IDs, dominant plane, plane records, stable radiance, guides) and the specular hit distance are the oracle's bit
    for bit; the noisy radiance the FILL pass deposits differs on a few paths in a thousand (libdevice vs glibc sin/cos/pow in the BSDF sampling)."""
    from rtxpt_b200 import scene_builder as sb
    g, g2, r, W, H = _run_pair(product, oracle, True)
    assert np.array_equal(g["header"], r["header"])
    ys, xs = np.mgrid[0:H, 0:W]
    for plane in range(3):
        v = r["header"][plane] != INVALID
        a = g["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]; b = r["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]
        for f in a.dtype.names:
            if f == "PackedNoisyRadianceAndSpecAvg": assert (a[f] == b[f]).all(-1).mean() > 0.995, (plane, f)
            elif a[f].dtype.kind == "u": assert np.array_equal(a[f], b[f]), (plane, f)             # packed words: identical
            else: assert np.allclose(a[f], b[f], rtol=1e-6, atol=1e-6, equal_nan=True), (plane, f)  # ray origin / direction / lengths (+inf marks a miss on both sides)
    for k in ("stable_radiance", "depth", "motion", "throughput", "spec_hit_t"): assert np.array_equal(g[k], r[k]), k
    d = np.abs(g["merged"] - r["merged"])
    assert (d == 0).all(-1).mean() > 0.995 and abs(g["merged"].mean() - r["merged"].mean()) < 1e-3 * r["merged"].mean()
    assert all(g[k].tobytes() == g2[k].tobytes() for k in g)                     # replay: bit-identical


@pytest.mark.gpu
def test_realtime_default_build_decomposes_like_the_oracle(product, oracle):
    """FMA / fast-math build: same decomposition (planes 0 and 2 identical, plane 1 except where the glass box's bottom face and the floor are hit at the
    same distance and ulp-level origin differences decide which comes first), same stable radiance, same image within noise."""
    from rtxpt_b200 import scene_builder as sb
    g, g2, r, W, H = _run_pair(product, oracle, False)
    assert np.array_equal(g["header"][0], r["header"][0]) and np.array_equal(g["header"][2], r["header"][2])
    assert (g["header"][1] == r["header"][1]).mean() > 0.98
    same = (g["header"][:3] == r["header"][:3]).all(0)
    ys, xs = np.nonzero(same)
    for plane in range(3):
        v = r["header"][plane][ys, xs] != INVALID
        a = g["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]; b = r["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]
        assert np.array_equal(a["VertexIndexAndRoughness"], b["VertexIndexAndRoughness"]) and (a["DenoiserPackedBSDFEstimate"] == b["DenoiserPackedBSDFEstimate"]).mean() > 0.97
        fin = np.isfinite(b["SceneLength"]); assert np.array_equal(np.isfinite(a["SceneLength"]), fin)
        assert np.allclose(a["SceneLength"][fin], b["SceneLength"][fin], rtol=1e-5) and np.allclose(a["RayDir"][fin], b["RayDir"][fin], atol=1e-3)
    assert (g["stable_radiance"] == r["stable_radiance"]).mean() > 0.999
    assert np.isclose(g["spec_hit_t"], r["spec_hit_t"], rtol=1e-3, atol=1e-3).mean() > 0.99
    assert np.isclose(g["depth"], r["depth"], rtol=2e-3, atol=1e-3).mean() > 0.98
    assert abs(g["merged"].mean() - r["merged"].mean()) < 0.03 * r["merged"].mean()
    assert all(g[k].tobytes() == g2[k].tobytes() for k in g)


def _same_headers(g, r, strict):
    """Pixels whose decomposition agrees.  Header words 0..2 are branch IDs (integers); word 3 is the first hit's ray length as float bits with the dominant plane index in its two
    low bits (StablePlanes.hlsli StoreFirstHitRayLengthAndClearDominantToZero): identical bits in the strict build, the length within a few ulp in the fast one."""
    if strict: return (g["header"] == r["header"]).all(0)
    la, lb = (g["header"][3] & 0xFFFFFFFC).view(np.float32), (r["header"][3] & 0xFFFFFFFC).view(np.float32)
    return (g["header"][:3] == r["header"][:3]).all(0) & ((g["header"][3] & 3) == (r["header"][3] & 3)) & np.isclose(la, lb, rtol=1e-5, atol=0)


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_build_pass_matches_oracle(product, oracle, strict):
    from rtxpt_b200 import scene_builder as sb
    W = H = 96
    c, o, cam, consts = _setup(product, oracle, strict, W, H)
    for kw in (dict(), dict(active_planes=2), dict(allow_psr=False), dict(max_vertex_depth=2)):
        rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1, **kw)
        c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize()
        g = c.readback_realtime(); r = o.render_realtime(rt)
        same = _same_headers(g, r, strict)
        assert same.mean() > (0.998 if strict else 0.98), (kw, same.mean())            # fast build: the glass box's bottom face and the floor are hit at the same distance, ulp-level origin differences decide which comes first (measured 0.988)
        ys, xs = np.nonzero(same)
        for plane in range(3):
            valid = r["header"][plane][ys, xs] != INVALID
            a = g["planes"][sb.generic_ts_address(xs[valid], ys[valid], plane, W, H)]; b = r["planes"][sb.generic_ts_address(xs[valid], ys[valid], plane, W, H)]
            if not len(a): continue
            assert (a["VertexIndexAndRoughness"] >> 16 == b["VertexIndexAndRoughness"] >> 16).all()
            fin = np.isfinite(b["SceneLength"])
            assert (np.isfinite(a["SceneLength"]) == fin).all()
            tol = 2e-6 if strict else 2e-4
            for f in ("RayOrigin", "RayDir", "SceneLength", "LastRayTCurrent"):
                x, y = a[f][fin], b[f][fin]
                assert np.allclose(x, y, rtol=tol, atol=tol * 10), (kw, plane, f, np.abs(x - y).max())
            for f in ("PackedThpAndMVs", "DenoiserPackedBSDFEstimate"):
                for xa, xb in zip(_halves(a[f]), _halves(b[f])):
                    if strict: assert np.allclose(xa, xb, rtol=4e-3, atol=1e-3), (kw, plane, f)
                    else:
                        # fast build: where the glass box's bottom face and the floor are hit at the same distance, ulp-level origin differences decide which surface the plane ends on
                        # (a share of plane 1's pixels with max_vertex_depth = 2); the estimate is compared where both sides ended on the same kind of surface
                        surface = a["VertexIndexAndRoughness"] == b["VertexIndexAndRoughness"]
                        assert surface.mean() > 0.75 and np.isclose(xa[surface], xb[surface], rtol=4e-3, atol=1e-3).mean() > 0.99, (kw, plane, f, surface.mean())
                if strict: assert (a[f] == b[f]).mean() > 0.99, (kw, plane, f, (a[f] == b[f]).mean())
            na = a["PackedNormal"]; nb = b["PackedNormal"]
            assert (np.abs((na & 0xFFFF).astype(np.int64) - (nb & 0xFFFF)) <= 8).mean() > 0.999 and (np.abs((na >> 16).astype(np.int64) - (nb >> 16)) <= 8).mean() > 0.999
        # stable radiance and the dominant plane's guides
        sa, sb_ = g["stable_radiance"].astype(np.float32), r["stable_radiance"].astype(np.float32)
        assert np.allclose(sa[same], sb_[same], rtol=2e-3, atol=1e-3)
        if strict: assert (g["stable_radiance"][same] == r["stable_radiance"][same]).all(-1).mean() > 0.995
        assert np.allclose(g["depth"][same], r["depth"][same], rtol=1e-5, atol=1e-6) and (g["throughput"][same] == r["throughput"][same]).mean() > 0.99
        assert np.allclose(g["motion"][same].astype(np.float32), r["motion"][same].astype(np.float32), atol=2e-3)
    c.close(); o.close()


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_fill_pass_and_merge_match_oracle(product, oracle, strict):
    from rtxpt_b200 import scene_builder as sb
    W = H = 96
    c, o, cam, consts = _setup(product, oracle, strict, W, H)
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=3)
    c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize()
    g = c.readback_realtime(); r = o.render_realtime(rt)
    same = _same_headers(g, r, strict)
    assert same.mean() > (0.998 if strict else 0.98)
    d = np.abs(g["merged"] - r["merged"])[same]; scale = np.maximum(r["merged"][same], 0.05)
    if strict:
        assert (d == 0).all(-1).mean() > 0.97, (d == 0).all(-1).mean()                # paths whose every decision agrees give the same fp16 sums
        assert np.percentile(d / scale, 99.5) < 0.05
    else:
        assert (d / scale < 0.02).all(-1).mean() > 0.9 and abs(g["merged"].mean() - r["merged"].mean()) < 1.5e-2 * r["merged"].mean()       # 3 sub-samples of a 96 x 96 frame
    # per-plane noisy radiance words and the specular hit distance
    ys, xs = np.nonzero(same)
    for plane in range(3):
        valid = r["header"][plane][ys, xs] != INVALID
        a = g["planes"][sb.generic_ts_address(xs[valid], ys[valid], plane, W, H)]["PackedNoisyRadianceAndSpecAvg"]
        b = r["planes"][sb.generic_ts_address(xs[valid], ys[valid], plane, W, H)]["PackedNoisyRadianceAndSpecAvg"]
        if strict and len(a): assert (a == b).all(-1).mean() > 0.96, (plane, (a == b).all(-1).mean())
    assert np.allclose(g["spec_hit_t"][same], r["spec_hit_t"][same], rtol=1e-3, atol=1e-3) or (np.isclose(g["spec_hit_t"][same], r["spec_hit_t"][same], rtol=1e-3, atol=1e-3).mean() > 0.995)
    c.close(); o.close()


@unverified
def test_realtime_invariants(product):
    """Size-independent properties at a larger frame: determinism, BUILD independent of the sub-sample count, the merged frame equals stable radiance plus
    the planes' noisy radiance, nothing left enqueued, and realtime frames average to the reference-mode image."""
    from rtxpt_b200 import scene_builder as sb, scenes
    W, H = 320, 200
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=4); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=2)
    c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize(); a = c.readback_realtime()
    c.path_trace_realtime(True); c.synchronize(); b = c.readback_realtime()
    for k in a: assert a[k].tobytes() == b[k].tobytes(), k
    hd = a["header"]
    assert (hd[0] != INVALID).all() and (hd[:3] != 0xFFFFFFFE).all() and (hd[:3] != 0).all()
    ys, xs = np.mgrid[0:H, 0:W]
    total = a["stable_radiance"][..., :3].astype(np.float32)
    for plane in range(3):
        w = a["planes"][sb.generic_ts_address(xs, ys, plane, W, H)]["PackedNoisyRadianceAndSpecAvg"]
        rgb = np.stack([(w[..., 0] & 0xFFFF), (w[..., 0] >> 16), (w[..., 1] & 0xFFFF)], -1).astype(np.uint16).view(np.float16).astype(np.float32)
        total = total + np.where((hd[plane] != INVALID)[..., None], rgb, 0)
    assert np.array_equal(total.astype(np.float16), a["merged"].astype(np.float16))
    rt1 = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1)
    c.set_realtime(rt1); c.path_trace_realtime(True); c.synchronize(); one = c.readback_realtime()
    assert np.array_equal(one["header"], a["header"]) and np.array_equal(one["stable_radiance"], a["stable_radiance"])
    # convergence to reference mode
    acc = np.zeros((H, W, 3), np.float64); frames = 8
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=4))
    for f in range(frames):
        consts.sampleBaseIndex = f * 4; c.set_constants(consts); c.path_trace_realtime(True); c.synchronize(); acc += c.readback_output_color()[..., :3].astype(np.float32)
    acc /= frames
    consts.sampleBaseIndex = 0; c.set_constants(consts); c.reset_accumulation(); c.path_trace(0, 32, True); c.synchronize()
    ref = c.readback_accumulated()[..., :3]
    assert abs(acc.mean() - ref.mean()) < 0.02 * ref.mean(), (acc.mean(), ref.mean())
    c.close()


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_denoiser_interface_matches_oracle(product, oracle, strict):
    """Row a18, RTXPT's side: NRD inputs prepared per plane and the final merge (here with the identity denoiser) against the oracle."""
    from rtxpt_b200 import scene_builder as sb
    W = H = 96
    c, o, cam, consts = _setup(product, oracle, strict, W, H)
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=2)
    c.set_realtime(rt); c.path_trace_realtime(False); c.synchronize()
    g = c.readback_realtime(); r = o.render_realtime(rt)
    k = sb.make_denoiser_constants(cam, suppress_primary_indirect_specular_k=0.4)
    d = o.new_denoiser_targets()
    same = _same_headers(g, r, strict)
    for i, plane in enumerate((2, 1, 0)):
        c.denoiser_prepare_inputs(plane, i == 0, k); c.synchronize(); gi = c.readback_denoiser_inputs()
        o.denoiser_prepare_inputs(rt, k, r, d, plane, i == 0)
        assert np.array_equal(gi["view_z"][same] < 1e30, d["view_z"][same] < 1e30)
        surf = same & (d["view_z"] < 1e30)
        assert np.allclose(gi["view_z"][surf], d["view_z"][surf], rtol=1e-5)
        assert (gi["normal_roughness"][surf] == d["normal_roughness"][surf]).mean() > 0.99 and (np.array_equal(gi["motion"][surf], d["motion"][surf]) if strict else np.allclose(gi["motion"][surf].astype(np.float32), d["motion"][surf].astype(np.float32), atol=1e-3))
        dm = np.abs(gi["disocclusion_mix"][surf].astype(int) - d["disocclusion_mix"][surf]) <= 1
        assert dm.all() if strict else dm.mean() > 0.9, dm.mean()          # fast build: same coincident-surface pixels as in test_build_pass_matches_oracle
        for key in ("diff", "spec"):
            a, b = gi[key][surf].astype(np.float32), d[key][surf].astype(np.float32)
            assert np.isclose(a, b, rtol=2e-2, atol=2e-3).all(-1).mean() > (0.97 if strict else 0.9), key
        c.denoiser_final_merge(plane); o.denoiser_final_merge(rt, r, d, plane, d["diff"].copy(), d["spec"].copy())
    c.synchronize()
    out = c.readback_output_color().astype(np.float32); ref = d["output"].astype(np.float32)
    assert np.isclose(out[same], ref[same], rtol=2e-2, atol=4e-3).all(-1).mean() > (0.97 if strict else 0.9)
    c.close(); o.close()


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_realtime_city_matches_oracle(product, oracle, strict):
    """Textured, environment-lit scene with NEE-AT proxies, alpha-tested foliage and glass opted into the decomposition."""
    from rtxpt_b200 import scene_builder as sb, scenes
    from test_oracle_realtime import _opt_glass_into_decomposition
    W, H = 160, 90
    scene, cam = scenes.city_block(target_triangles=120000, width=W, height=H, texture_size=128, n_textures=6, n_materials=64)
    _opt_glass_into_decomposition(scene)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2)
    c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime(); r = o.render_realtime(rt)
    same = (g["header"][:3] == r["header"][:3]).all(0)
    assert same.mean() > 0.995
    assert (g["stable_radiance"][same] == r["stable_radiance"][same]).all(-1).mean() > (0.99 if strict else 0.95)
    d = np.abs(g["merged"] - r["merged"])[same]; scale = np.maximum(r["merged"][same], 0.05)
    assert (d / scale < 0.05).all(-1).mean() > (0.95 if strict else 0.85)          # texture filtering (TMU vs software) and transcendental differences change some paths
    assert abs(g["merged"].mean() - r["merged"].mean()) < 0.02 * r["merged"].mean()
    c.close(); o.close()


@pytest.mark.gpu
def test_config3_frame_split_over_two_ranks_equals_the_single_gpu_frame(product):
    """SURVEY §8e for BASELINE configs[2]: two contexts own interleaved 32x32 screen tiles of the frame (both on this GPU; the all-gather is a device copy) and run the recipe of
    include/rtxpt_b200.h - trace own tiles, exchange guides, per plane { prepare, exchange NRD inputs, ReBLUR on the whole frame, merge }, exchange the output colour, tone map.
    Without NEE-AT feedback every per-pixel step is deterministic and ReBLUR sees identical inputs: three consecutive frames are bit-identical to one context's frames,
    in what the denoiser received, what it returned, its history lengths and the tone-mapped image.  With feedback each rank adapts on its own tiles: same mean, finite."""
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S, realtime_mgpu as M
    W, H = 160, 128
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    k = sb.make_denoiser_constants(cam); tm = S.make_tone_mapping_params(op=5, auto_exposure=True)
    def make(rank, world):
        c = product.Context(max_sub_samples_per_launch=1, tile_rank=rank, tile_world=world, tile_size=32); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
        c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2)); return c
    one = make(0, 1); two = [make(0, 2), make(1, 2)]; group = M.LocalGroup(two)
    for f in range(3):
        consts.sampleBaseIndex = 2 * f
        for c in [one] + two: c.set_constants(consts)
        frame = sb.make_reblur_frame(cam, cam, frame_index=f)
        one.path_trace_realtime(False); one.denoise_realtime(k, frame); one.tone_map(tm); one.synchronize()
        moved = M.realtime_frame(group, k, frame, tm)
        for c in two: c.synchronize()
        ref = dict(inputs=one.readback_denoiser_inputs(), reblur=one.readback_reblur(), color=one.readback_output_color(), ldr=one.readback_ldr(), guides=one.readback_guides())
        for c in two:
            got = dict(inputs=c.readback_denoiser_inputs(), reblur=c.readback_reblur(), color=c.readback_output_color(), ldr=c.readback_ldr(), guides=c.readback_guides())
            for key in ("inputs", "reblur"):
                for name in ref[key]: assert ref[key][name].tobytes() == got[key][name].tobytes(), (f, key, name)
            assert ref["color"].tobytes() == got["color"].tobytes() and ref["ldr"].tobytes() == got["ldr"].tobytes(), f
            assert ref["guides"][0].tobytes() == got["guides"][0].tobytes()                 # depth: exchanged; motion / throughput stay per rank
        assert moved == 2 * (two[0].exchange_bytes(M.GUIDES) + 3 * two[0].exchange_bytes(M.NRD_INPUTS) + two[0].exchange_bytes(M.OUTPUT))
    # with NEE-AT feedback: each rank keeps its own reservoirs and global table
    consts.NEEATFeedback = 1; means = []
    for f in range(6):
        consts.sampleBaseIndex = 100 + 2 * f
        for c in [one] + two: c.set_constants(consts)
        frame = sb.make_reblur_frame(cam, cam, frame_index=3 + f)
        one.neeat_update_begin(); one.path_trace_realtime(False); one.denoise_realtime(k, frame); one.synchronize()
        M.realtime_frame(group, k, frame, None, feedback=True)
        for c in two: c.synchronize()
        a = one.readback_output_color()[..., :3].astype(np.float32); b = two[0].readback_output_color()[..., :3].astype(np.float32)
        assert np.isfinite(b).all() and two[0].readback_output_color().tobytes() == two[1].readback_output_color().tobytes()
        means.append((a.mean(), b.mean()))
    m = np.asarray(means)
    assert abs(m[:, 1].mean() / m[:, 0].mean() - 1) < 0.03, means
    for c in [one] + two: c.close()
