"""GPU: approximate light-vs-BSDF MIS (RtxptPathTracerConstants::useApproximateMIS = 1, the AMIS instantiations of k_shade and k_rt_shade) through the C ABI, against the CPU oracle
with the same switch (oracle/amis.mk, tests/oracle_amis_lib.py).  Bars as for full MIS: the strict (IEEE) build traces the oracle's rays and is bit-identical on nearly every pixel, the default build meets the tolerances of
test_gpu_parity.py; realtime mode's planes and radiance as in test_gpu_realtime.py; NEE-AT's feedback state bit for bit as in test_gpu_neeat.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle():
    """the approximate-MIS oracle; with useApproximateMIS = 0 it is the full-MIS oracle"""
    import oracle_amis_lib
    oracle_amis_lib.build()
    return oracle_amis_lib.oracle


@pytest.fixture(scope="module", params=["fast", "strict"])
def ctx(product, request):
    c = product.Context(max_sub_samples_per_launch=4, strict=(request.param == "strict"))
    c.variant = request.param
    yield c
    c.close()


def _reference_pair(ctx, oracle, scene, consts, spp):
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.reset_accumulation()
    o = oracle.Oracle(scene); o.set_constants(consts)
    ctx.path_trace(0, spp, True); ctx.synchronize(); img = ctx.readback_accumulated(); st = ctx.stats()
    acc, n, _, _, ost = o.render(0, spp); o.close()
    return img, st, acc, ost


@pytest.mark.parametrize("full", [1, 3])
def test_cornell_approximate_mis_parity(product, ctx, oracle, full):
    """Cornell box with its emissive quad, a sphere light with proxy geometry (the analytic-proxy MIS), a spot light and the sky behind the open side (the environment miss), 192 x 192,
    2 spp in one launch, 3 bounces; NEEFullSamples 1 and 3 (the multi-sample AMIS kernel)."""
    from rtxpt_b200 import scene_builder as sb, scenes
    from rtxpt_b200.imageio import per_pixel_l2
    b = scenes.cornell_builder(analytic_lights=True); b.set_env_cube(scenes.sky_cube(64, sun_intensity=4.0)); scene = b.build()
    cam = sb.bridge_camera(192, 192, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    consts = sb.make_constants(192, 192, cam, bounce_count=3, diffuse_bounce_count=3, env_enabled=True, nee_full=full, approximate_mis=True)
    c = product.Context(max_sub_samples_per_launch=2 * full, strict=(ctx.variant == "strict"))       # both sub-samples in one launch: the ray counts are those of the call
    img, st, acc, ost = _reference_pair(c, oracle, scene, consts, 2)
    d = np.abs(img[..., :3] - acc[..., :3])
    if ctx.variant == "strict":
        assert st.scatterRays == ost.scatterRays and st.shadowRays == ost.shadowRays
        assert (d.max(-1) == 0).mean() > 0.99 and per_pixel_l2(img, acc) < 1e-6
    else:
        assert abs(int(st.scatterRays) - int(ost.scatterRays)) <= 1e-3 * ost.scatterRays and abs(int(st.shadowRays) - int(ost.shadowRays)) <= 1e-3 * ost.shadowRays
        assert per_pixel_l2(img, acc) < 1e-4
    # the switch reaches the kernels: the same frame with full MIS is another image
    consts.useApproximateMIS = 0
    c.set_constants(consts); c.reset_accumulation(); c.path_trace(0, 2, True); c.synchronize()
    assert not np.array_equal(c.readback_accumulated(), img)
    c.close()


def test_city_approximate_mis_parity(ctx, oracle, small_city):
    """The small city (environment quad-tree lights, emissive triangles, textures, alpha test, glass, firefly filter, roulette), 1 spp: the bars of
    test_city_image_parity_and_accumulation; the strict build also traces the oracle's rays to 2e-3."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = small_city
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, approximate_mis=True)
    img, st, acc, ost = _reference_pair(ctx, oracle, scene, consts, 1)
    assert abs(int(st.scatterRays) - int(ost.scatterRays)) < 2e-3 * ost.scatterRays
    rel = np.abs(img[..., :3] - acc[..., :3]) / (np.abs(acc[..., :3]) + 1e-2)
    assert (rel.max(-1) < 5e-2).mean() > 0.995
    assert per_pixel_l2(img, acc) < 1e-3


@pytest.mark.parametrize("full", [1, 3])
def test_realtime_approximate_mis_strict_build_is_the_oracle(product, oracle, full):
    """Realtime mode without feedback, strict build, NEEFullSamples 1 and 3: the BUILD pass's headers, plane records and stable radiance are the oracle's bit for bit, and the noisy
    radiance the AMIS FILL pass deposits in the planes agrees on nearly every plane (as in test_gpu_realtime).  The sky seen through the mirror makes plane 1 the least exact: measured on
    an H100, 0.995 / 0.993 of its 761 pixels with N = 1 / 3 (0.989 with full MIS on the same scene)."""
    from rtxpt_b200 import scene_builder as sb, scenes
    W = H = 96
    b = scenes.cornell_builder(delta_surfaces=True); b.set_env_cube(scenes.sky_cube(64, sun_intensity=4.0)); scene = b.build()
    cam = sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3, env_enabled=True, nee_full=full, approximate_mis=True)
    c = product.Context(max_sub_samples_per_launch=1, strict=True); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=2)
    c.set_realtime(rt); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    r = o.render_realtime(rt)
    c.close(); o.close()
    assert np.array_equal(g["header"], r["header"])
    ys, xs = np.mgrid[0:H, 0:W]
    for plane in range(3):
        v = r["header"][plane] != 0xFFFFFFFF
        a = g["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]; bb = r["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]
        for f in a.dtype.names:
            if f == "PackedNoisyRadianceAndSpecAvg": assert (a[f] == bb[f]).all(-1).mean() > 0.99, (plane, f)
            elif a[f].dtype.kind == "u": assert np.array_equal(a[f], bb[f]), (plane, f)
            else: assert np.allclose(a[f], bb[f], rtol=1e-6, atol=1e-6, equal_nan=True), (plane, f)
    assert np.array_equal(g["stable_radiance"], r["stable_radiance"])
    assert ((g["merged"] == r["merged"]).all(-1)).mean() > 0.995


def test_realtime_approximate_mis_neeat_feedback(product, oracle):
    """RTXPT's realtime default: NEE-AT with temporal feedback and approximate MIS, strict build, five frames of the light gallery.  Both sides run their own frames; each frame the
    GPU starts from the reservoirs the oracle's path tracer filled, so that its feedback passes see the same inputs: reservoirs, usage counters and proxy table bit for bit after
    update_begin (update_end reprojects through the depth guide, which agrees to ulps only: test_gpu_neeat.py), the BUILD pass's headers bit for bit, and the reservoirs the
    GPU's own AMIS FILL pass fills pick the oracle's light in nearly every pixel."""
    from rtxpt_b200 import scene_builder as sb, scenes
    W, H = 90, 58
    scene, cam = scenes.light_gallery(W, H, bays=7)
    consts = sb.make_constants(W, H, cam, bounce_count=2, diffuse_bounce_count=2, approximate_mis=True); consts.NEEATFeedback = 1; consts.NEEATImportanceBoost = 3
    c = product.Context(max_sub_samples_per_launch=1, strict=True); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam)); o.neeat_reset()
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=2, sub_samples=1); c.set_realtime(rt)
    n_lights = int(o.neeat_raw(12, np.uint32, 1)[0]); P = W * H

    def same_state(stage):
        co, cp = o.neeat_raw(8, np.uint32, 8), c.neeat_raw(8, np.uint32, 8)
        assert np.array_equal(co, cp), (stage, co, cp)
        for what, n, name in ((0, P, "feedback weight"), (1, P, "feedback candidate"), (7, n_lights, "proxy counters"), (11, int(co[4]), "proxy table")):
            a, b = o.neeat_raw(what, np.uint32, n), c.neeat_raw(what, np.uint32, n)
            assert len(a) == len(b) == n and np.array_equal(a, b), (stage, name, int((a != b).sum()))

    agree = []
    for f in range(5):
        consts.sampleBaseIndex = f; c.set_constants(consts); o.set_constants(consts)
        if f > 0: c.neeat_set_feedback(o.neeat_raw(0, np.float32, P), o.neeat_raw(1, np.uint32, P))
        o.neeat_update_begin(); c.neeat_update_begin(); c.synchronize(); same_state("begin")
        r = o.render_realtime(rt); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
        assert np.array_equal(g["header"], r["header"])
        agree.append(float((c.neeat_raw(1, np.uint32, P) == o.neeat_raw(1, np.uint32, P)).mean()))
    c.close(); o.close()
    assert min(agree) > 0.9, agree                    # the reservoirs this frame's FILL pass filled: the same light picked in nearly every pixel


def test_reference_mode_neeat_feedback_runs_the_approximate_kernel(product):
    """Reference mode with NEE-AT feedback (the NEE-AT instantiation of k_shade with AMIS): update_begin / update_end on the guides of the previous frame, eight frames; the images are
    finite, and the same frames with full MIS are other images of the same mean (within 3 %)."""
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    W, H = 112, 72
    scene, cam = scenes.light_gallery(W, H, bays=10)

    def frames(approx):
        consts = sb.make_constants(W, H, cam, bounce_count=2, diffuse_bounce_count=2, approximate_mis=approx)
        c = product.Context(max_sub_samples_per_launch=4, flags=S.CFG_EXPORT_GUIDES); c.upload_scene(scene); c.set_view(sb.world_to_clip(cam))
        consts.NEEATFeedback = 0; c.set_constants(consts); c.path_trace(0, 1, False); c.synchronize()        # a first frame leaves depth / motion guides behind
        consts.NEEATFeedback = 1; out = []
        for f in range(8):
            consts.sampleBaseIndex = 2 * f; c.set_constants(consts); c.neeat_update_begin(); c.neeat_update_end()
            c.path_trace(0, 2, False); c.synchronize(); out.append(c.readback_output_color()[..., :3].astype(np.float32))
        c.close()
        return np.stack(out)
    a, f = frames(True), frames(False)
    assert np.isfinite(a).all() and not np.array_equal(a, f)
    assert abs(a.mean() / f.mean() - 1) < 0.03, (a.mean(), f.mean())


def test_approximate_mis_field_is_validated(product, cornell):
    """useApproximateMIS 2 and 0xFFFFFFFF are refused with RTXPT_ERR_INVALID_ARGUMENT and leave the constants as they were: the next frame renders as the frame before."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.lib import RtxptError
    scene, cam = cornell
    c = product.Context(max_sub_samples_per_launch=2)
    c.upload_scene(scene)
    consts = sb.make_constants(128, 128, cam, bounce_count=2, diffuse_bounce_count=2, approximate_mis=True)

    def frame():
        c.reset_accumulation(); c.path_trace(0, 2, True); c.synchronize()
        return c.readback_accumulated()
    c.set_constants(consts); before = frame()
    for bad in (2, 0xFFFFFFFF):
        k = sb.make_constants(128, 128, cam, bounce_count=2, diffuse_bounce_count=2); k.useApproximateMIS = bad
        with pytest.raises(RtxptError, match="error -1"):
            c.set_constants(k)
    after = frame()
    assert np.array_equal(before, after) and np.isfinite(after).all() and after[..., :3].mean() > 0
    c.close()
