"""GPU: stochastic texture filtering against the oracle with pt_stf.h applied (oracle/stf.mk, tests/oracle_stf_lib.py), both libraries.  The oracle draws the vertex's u with its
own sample generator, picks texels with its own restatement of the RTXTF header and reads them from the host texture data; the product fetches them through point-filtered texture
objects.  Bars as in test_gpu_approximate_mis.py / test_gpu_parity.py: the strict (IEEE) build traces the oracle's rays and is bit-identical on nearly every pixel, the default build
meets the tolerances of the image-parity tests.  Also: the 2-way tile split, and a 1024-spp STF-Linear accumulation against hardware trilinear on an albedo-only scene."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
FILTERS = [0, 1, 2, 3]


@pytest.fixture(scope="module")
def oracle():
    import oracle_stf_lib
    oracle_stf_lib.build()
    return oracle_stf_lib


def _checker(rng, w, h, srgb_scale=255):
    img = np.zeros((h, w, 4), np.uint8)
    img[..., :3] = rng.integers(0, srgb_scale + 1, (h, w, 3)); img[..., 3] = 255
    return img


def textured_cornell(delta_surfaces=False, albedo_only=False, srgb=True):
    """cornell_builder's room with textures on every material slot RTXPT samples: odd and power-of-two sizes, sRGB albedo, linear ORM and normal maps, an emissive texture on the lamp"""
    from rtxpt_b200 import scenes
    rng = np.random.default_rng(7)
    b = scenes.cornell_builder(delta_surfaces=delta_surfaces)
    alb = [b.add_texture(_checker(rng, s, s), srgb=srgb) for s in (37, 64, 13)]
    mats = b.materials
    for i, m in enumerate(mats[:3]):                                                         # white, red, green
        m.base_texture = alb[i]
        if not albedo_only:
            orm = _checker(rng, 32, 32); orm[..., 1] = np.maximum(orm[..., 1], 60)
            m.orm_texture = b.add_texture(orm, srgb=False)
            nrm = np.zeros((16, 16, 4), np.uint8); nrm[..., 0:2] = rng.integers(100, 156, (16, 16, 2)); nrm[..., 2] = 230; nrm[..., 3] = 255
            m.normal_texture = b.add_texture(nrm, srgb=False)
    if not albedo_only:
        mats[3].emissive_texture = b.add_texture(_checker(rng, 8, 8), srgb=srgb)
    return b.build()


def _camera(W, H):
    from rtxpt_b200 import scene_builder as sb
    return sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)


def _pair(product, oracle, scene, consts, strict, filt, spp):
    c = product.Context(max_sub_samples_per_launch=spp, strict=strict)
    c.upload_scene(scene); c.set_constants(consts); c.set_texture_filtering(True, filt, 0, 0.3)
    c.path_trace(0, spp, True); c.synchronize(); img = c.readback_accumulated(); st = c.stats()
    c.set_texture_filtering(False); c.reset_accumulation(); c.path_trace(0, spp, True); c.synchronize(); off = c.readback_accumulated(); c.close()
    o = oracle.oracle.Oracle(scene); o.set_constants(consts); oracle.set_texture_filtering(o, True, filt, 0.3)
    acc, n, _, _, ost = o.render(0, spp); o.close()
    return img, st, acc, ost, off


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("filt", FILTERS)
@pytest.mark.parametrize("srgb", [False, True])
def test_cornell_stf_parity(product, oracle, strict, filt, srgb):
    """Textured Cornell box, 128 x 128, 2 spp in one launch, 3 bounces, every filter: the bars of test_cornell_approximate_mis_parity with UNORM textures; the filter reaches the
    kernels.  With sRGB textures the texture unit's sRGB decode of the fetched texel and the oracle's table are not the same floats, so the strict build is held to the default
    build's bars there (measured on an H100: ray counts within 5 of 91 000)."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    W = H = 128
    scene = textured_cornell(srgb=srgb)
    consts = sb.make_constants(W, H, _camera(W, H), bounce_count=3, diffuse_bounce_count=3)
    img, st, acc, ost, off = _pair(product, oracle, scene, consts, strict, filt, 2)
    d = np.abs(img[..., :3] - acc[..., :3])
    if strict and not srgb:
        assert st.scatterRays == ost.scatterRays and st.shadowRays == ost.shadowRays
        assert (d.max(-1) == 0).mean() > 0.99 and per_pixel_l2(img, acc) < 1e-6, ((d.max(-1) == 0).mean(), per_pixel_l2(img, acc))
    else:
        assert abs(int(st.scatterRays) - int(ost.scatterRays)) <= 1e-3 * ost.scatterRays
        assert per_pixel_l2(img, acc) < 1e-4, per_pixel_l2(img, acc)
    assert not np.array_equal(img, off)


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("filt", [1, 3])
def test_city_stf_parity(product, oracle, small_city, strict, filt):
    """The small city (sRGB albedo and linear ORM textures at 128 x 128 with full chains, alpha test, glass, environment), 1 spp: the bars of test_city_approximate_mis_parity"""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = small_city
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0)
    img, st, acc, ost, off = _pair(product, oracle, scene, consts, strict, filt, 1)
    assert abs(int(st.scatterRays) - int(ost.scatterRays)) < 2e-3 * ost.scatterRays
    rel = np.abs(img[..., :3] - acc[..., :3]) / (np.abs(acc[..., :3]) + 1e-2)
    assert (rel.max(-1) < 5e-2).mean() > 0.995
    assert per_pixel_l2(img, acc) < 1e-3
    assert not np.array_equal(img, off)


@pytest.mark.parametrize("filt", [1, 2])
def test_realtime_stf_strict_build_is_the_oracle(product, oracle, filt):
    """Realtime BUILD and FILL with STF, strict build, textured Cornell box (UNORM textures) with a mirror and glass: the bars of test_realtime_approximate_mis_strict_build_is_the_oracle"""
    from rtxpt_b200 import scene_builder as sb, scenes
    W = H = 96
    scene = textured_cornell(delta_surfaces=True, srgb=False)
    cam = _camera(W, H)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=True); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    c.set_texture_filtering(True, filt, 0, 0.3)
    o = oracle.oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam)); oracle.set_texture_filtering(o, True, filt, 0.3)
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


@pytest.mark.parametrize("strict", [False, True])
def test_tile_split_with_stf(product, small_city, strict):
    """a 2-way tile partition (two contexts on one GPU) + pack / unpack reassembles the single-context STF frame bit for bit, as test_determinism_batching_and_tiles does without STF"""
    import torch
    from rtxpt_b200 import scene_builder as sb
    scene, cam = small_city
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, env_enabled=True, firefly_threshold=5000.0)
    def render(ctx):
        ctx.upload_scene(scene); ctx.set_constants(consts); ctx.set_texture_filtering(True, 2, 0, 0.3); ctx.reset_accumulation(); ctx.path_trace(0, 4)
        return ctx.readback_accumulated()
    a = product.Context(max_sub_samples_per_launch=4, strict=strict); ia = render(a); a.close()
    parts = [product.Context(max_sub_samples_per_launch=4, tile_rank=r, tile_world=2, tile_size=32, strict=strict) for r in range(2)]
    for p in parts: render(p)
    padded = parts[0].tile_layout()[1]
    gathered = torch.zeros((2 * padded, 4), dtype=torch.float32, device="cuda")
    for r, p in enumerate(parts):
        p.synchronize(); p.pack_owned(gathered[r * padded:(r + 1) * padded].data_ptr()); p.synchronize()
    parts[0].unpack_all(gathered.data_ptr()); parts[0].synchronize()
    assert np.array_equal(parts[0].readback_accumulated(), ia)
    for p in parts: p.close()


def test_stf_linear_converges_to_trilinear(product):
    """Albedo-only diffuse Cornell box (textured albedo, roughness 1, no other texture), 64 x 64, 1024 spp, default build: STF-Linear picks average to the trilinear texel value, and a
    vertex's albedo enters the path linearly, so the two accumulations agree up to sampling noise and the TMU's 8-bit filter weights.  Bar (measured): image mean within 0.5 %,
    8 x 8 block means within 3 %."""
    from rtxpt_b200 import scene_builder as sb
    W = H = 64
    scene = textured_cornell(albedo_only=True)
    consts = sb.make_constants(W, H, _camera(W, H), bounce_count=4, diffuse_bounce_count=4)
    imgs = []
    for on in (False, True):
        c = product.Context(max_sub_samples_per_launch=16); c.upload_scene(scene); c.set_constants(consts); c.set_texture_filtering(on, 1, 0, 0.3)
        for k in range(64): c.path_trace(16 * k, 16, True)
        c.synchronize(); imgs.append(c.readback_accumulated()[..., :3].astype(np.float64)); c.close()
    tri, stf = imgs
    mean_rel = abs(stf.mean() / tri.mean() - 1)
    bt = tri.reshape(8, 8, 8, 8, 3).mean((1, 3)); bs = stf.reshape(8, 8, 8, 8, 3).mean((1, 3))
    lit = bt > 0.02 * bt.max()
    block_rel = np.abs(bs[lit] / bt[lit] - 1).max()
    assert mean_rel < 5e-3 and block_rel < 3e-2, (mean_rel, block_rel)
