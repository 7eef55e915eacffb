"""GPU: NEEFullSamples > 1 - several light samples per path vertex, each with its own shadow ray (PathTracerNEE.hlsli:277-346) - through the C ABI, against the CPU oracle's
HandleNEE loop.  The multi-sample shade appends one shadow record per valid sample and parks the sample's fp32 result in the vertex's NEE block; the shadow kernel marks the visible
samples and k_nee_resolve sums them in sample order with fp16 rounding after every add, before the one AccumulatePathRadiance."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["fast", "strict"])
def ctx(product, request):
    c = product.Context(max_sub_samples_per_launch=4, strict=(request.param == "strict"))
    c.variant = request.param
    yield c
    c.close()


@pytest.mark.parametrize("full", [2, 3, 8])
def test_cornell_c1_multi_sample_parity(ctx, oracle, cornell, full):
    """Cornell box 256x256, 1 spp, 2 bounces: the strict build traces the oracle's rays (scatter and shadow counts equal) and is bit-identical on more than 99.5 % of the
    pixels; the default build is held to the bars of test_cornell_c1_image_parity."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = cornell
    consts = sb.make_constants(256, 256, cam, bounce_count=2, diffuse_bounce_count=2, nee_full=full)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.reset_accumulation()
    o = oracle.Oracle(scene); o.set_constants(consts)
    ctx.path_trace(0, 1); img = ctx.readback_accumulated(); st = ctx.stats()
    acc, n, last, prim, ost = o.render(0, 1); o.close()
    assert ost.shadowRays > 1.5 * 256 * 256          # several samples per vertex were traced
    d = np.abs(img[..., :3] - acc[..., :3])
    if ctx.variant == "strict":
        assert st.scatterRays == ost.scatterRays and st.shadowRays == ost.shadowRays
        assert (d.max(-1) == 0).mean() > 0.995 and d.max() < 2e-2 and per_pixel_l2(img, acc) < 1e-7
    else:
        assert abs(int(st.scatterRays) - int(ost.scatterRays)) <= 1e-3 * ost.scatterRays and abs(int(st.shadowRays) - int(ost.shadowRays)) <= 1e-3 * ost.shadowRays
        rel = d / (np.abs(acc[..., :3]) + 1e-2)
        assert (rel.max(-1) < 2e-2).mean() > 0.998 and per_pixel_l2(img, acc) < 1e-4


@pytest.mark.parametrize("full", [2, 4])
def test_city_multi_sample_parity(ctx, oracle, small_city, full):
    """The small city (environment quad-tree lights, emissive triangles, textures, alpha test, glass, firefly filter, roulette), 1 spp: ray counts within 2e-3 of the
    oracle's, per-pixel L2 at most 1e-3."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = small_city
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee_full=full)
    ctx.upload_scene(scene); ctx.set_constants(consts); ctx.reset_accumulation()
    o = oracle.Oracle(scene); o.set_constants(consts)
    ctx.path_trace(0, 1); img = ctx.readback_accumulated(); st = ctx.stats()
    acc, n, _, _, ost = o.render(0, 1); o.close()
    assert abs(int(st.scatterRays) - int(ost.scatterRays)) <= 2e-3 * ost.scatterRays and abs(int(st.shadowRays) - int(ost.shadowRays)) <= 2e-3 * ost.shadowRays
    assert ost.shadowRays > 1.2 * W * H
    assert per_pixel_l2(img, acc) <= 1e-3


def test_analytic_lights_multi_sample_parity(product, ctx, oracle):
    """Sphere, spot and point lights next to the emissive triangles, NEEFullSamples = 3, 4 spp in one launch (12 / 3 sub-samples per launch: the ray counts of get_stats are
    those of the call, not extrapolated from its last launch)."""
    from rtxpt_b200 import scene_builder as sb, scenes
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = scenes.cornell_box(192, 192, analytic_lights=True)
    consts = sb.make_constants(192, 192, cam, bounce_count=3, diffuse_bounce_count=3, nee_full=3)
    c = product.Context(max_sub_samples_per_launch=12, strict=(ctx.variant == "strict"))
    c.upload_scene(scene); c.set_constants(consts)
    o = oracle.Oracle(scene); o.set_constants(consts)
    c.path_trace(0, 4, True); img = c.readback_accumulated(); st = c.stats(); c.close()
    acc, n, _, _, ost = o.render(0, 4); o.close()
    d = np.abs(img[..., :3] - acc[..., :3])
    if ctx.variant == "strict":
        assert st.scatterRays == ost.scatterRays and st.shadowRays == ost.shadowRays
        assert (d.max(-1) == 0).mean() > 0.99 and per_pixel_l2(img, acc) < 1e-6
    else:
        assert abs(int(st.shadowRays) - int(ost.shadowRays)) <= 1e-3 * ost.shadowRays and per_pixel_l2(img, acc) < 1e-4


@pytest.mark.parametrize("strict", [False, True])
def test_multi_sample_batch_and_tile_invariance(product, small_city, strict):
    """NEEFullSamples = 3: four sub-samples in one wavefront, four single launches and two launches of two give the same bits, and a 2-way tile partition reassembles the
    frame bit for bit."""
    import torch
    from rtxpt_b200 import scene_builder as sb
    scene, cam = small_city
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, env_enabled=True, firefly_threshold=5000.0, nee_full=3)

    def render(c, batches):
        c.upload_scene(scene); c.set_constants(consts); c.reset_accumulation()
        s = 0
        for n in batches:
            c.path_trace(s, n); s += n
        return c.readback_accumulated()
    a = product.Context(max_sub_samples_per_launch=12, strict=strict); b = product.Context(max_sub_samples_per_launch=1, strict=strict)     # 12 / 3: four sub-samples per launch
    ia = render(a, [4]); ib = render(b, [1, 1, 1, 1]); ic = render(a, [2, 2])
    assert a.stats().shadowRays > 0
    assert np.array_equal(ia, ib) and np.array_equal(ia, ic)
    a.close(); b.close()
    parts = [product.Context(max_sub_samples_per_launch=12, tile_rank=r, tile_world=2, tile_size=32, strict=strict) for r in range(2)]
    for p in parts:
        render(p, [4])
    padded = parts[0].tile_layout()[1]
    gathered = torch.zeros((2 * padded, 4), dtype=torch.float32, device="cuda")
    for r, p in enumerate(parts):
        p.synchronize(); p.pack_owned(gathered[r * padded:(r + 1) * padded].data_ptr()); p.synchronize()
    parts[0].unpack_all(gathered.data_ptr()); parts[0].synchronize()
    assert np.array_equal(parts[0].readback_accumulated(), ia)
    for p in parts:
        p.close()


@pytest.mark.parametrize("full", [2, 3])
def test_realtime_fill_multi_sample_strict_build_is_the_oracle(product, oracle, full):
    """Realtime mode without feedback (NEEATFeedback = 0), strict build: the BUILD pass's headers and plane records and the stable radiance are the oracle's bit for bit, and the
    noisy radiance the multi-sample FILL pass deposits in the planes agrees on nearly every plane (as in test_gpu_realtime)."""
    from rtxpt_b200 import scene_builder as sb, scenes
    W = H = 96
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3, nee_full=full)
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
        a = g["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]; b = r["planes"][sb.generic_ts_address(xs[v], ys[v], plane, W, H)]
        for f in a.dtype.names:
            if f == "PackedNoisyRadianceAndSpecAvg": assert (a[f] == b[f]).all(-1).mean() > 0.995, (plane, f)
            elif a[f].dtype.kind == "u": assert np.array_equal(a[f], b[f]), (plane, f)
            else: assert np.allclose(a[f], b[f], rtol=1e-6, atol=1e-6, equal_nan=True), (plane, f)
    assert np.array_equal(g["stable_radiance"], r["stable_radiance"])
    d = np.abs(g["merged"] - r["merged"])
    assert (d == 0).all(-1).mean() > 0.995


def test_full_samples_limits(product, cornell):
    """NEEFullSamples = 0 traces no shadow ray; 64 renders as 63 (the shader's min); 2 with NEE-AT feedback is refused with RTXPT_ERR_UNSUPPORTED and the context renders afterwards."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.lib import RtxptError
    scene, cam = cornell
    c = product.Context(max_sub_samples_per_launch=4)
    c.upload_scene(scene)

    def frame(full, **kw):
        consts = sb.make_constants(128, 128, cam, bounce_count=2, diffuse_bounce_count=2, nee_full=full, **kw)
        c.set_constants(consts); c.reset_accumulation(); c.path_trace(0, 2, True); c.synchronize()
        return c.readback_accumulated(), c.stats()
    img0, st0 = frame(0)
    assert st0.shadowRays == 0 and st0.scatterRays > 0 and np.isfinite(img0).all()
    img63, st63 = frame(63); img64, st64 = frame(64)
    assert np.array_equal(img63, img64) and st63.shadowRays == st64.shadowRays > 20 * 128 * 128
    consts = sb.make_constants(128, 128, cam, bounce_count=2, diffuse_bounce_count=2, nee_full=2)
    consts.NEEATFeedback = 1
    with pytest.raises(RtxptError, match="error -6"):
        c.set_constants(consts)
    img1, st1 = frame(1)
    assert np.isfinite(img1).all() and 0 < st1.shadowRays <= st1.scatterRays and img1[..., :3].mean() > 0
    c.close()
