"""GPU: stochastic texture filtering of the material fetches (rtxpt_b200_set_texture_filtering, the STF instantiations of k_shade and k_rt_shade), both libraries, on a small
textured city.  Off gives back the frames of a context that never enabled it, bit for bit; every refused description leaves the next frame unchanged; with STF on the frames are
deterministic, independent of how many sub-samples a launch batches, and each filter changes the textured image; the realtime BUILD / FILL passes run with it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
W, H = 192, 112


@pytest.fixture(scope="module")
def city():
    from rtxpt_b200 import scenes, scene_builder as sb
    scene, cam = scenes.city_block(target_triangles=40000, width=W, height=H, texture_size=64, n_textures=4, n_materials=32)
    return scene, cam, sb.make_constants(W, H, cam, bounce_count=3, diffuse_bounce_count=3)


def _frame(product, strict, city, spp=2, stf=None, batch=2, refused=()):
    scene, cam, consts = city
    c = product.Context(max_sub_samples_per_launch=batch, strict=strict)
    try:
        c.upload_scene(scene); c.set_constants(consts)
        if stf is not None: c.set_texture_filtering(**stf)
        for bad in refused:
            with pytest.raises(product.RtxptError) as e: c.set_texture_filtering(**bad)
            assert ("error %d" % (-6 if bad.get("magnification_method", 0) in range(1, 7) else -1)) in str(e.value), (bad, str(e.value))
        c.path_trace(0, spp, True); c.synchronize()
        return c.readback_accumulated()
    finally:
        c.close()


@pytest.mark.parametrize("strict", [False, True])
def test_disabled_is_never_enabled(product, city, strict):
    base = _frame(product, strict, city)
    scene, cam, consts = city
    c = product.Context(max_sub_samples_per_launch=2, strict=strict)
    c.upload_scene(scene); c.set_constants(consts)
    c.set_texture_filtering(True, 1); c.path_trace(0, 2, True); c.synchronize(); on = c.readback_accumulated()
    c.set_texture_filtering(False); c.reset_accumulation(); c.path_trace(0, 2, True); c.synchronize(); off = c.readback_accumulated()
    c.close()
    assert off.tobytes() == base.tobytes()
    assert on.tobytes() != base.tobytes()


@pytest.mark.parametrize("strict", [False, True])
def test_refused_descriptions_leave_the_frame(product, city, strict):
    cubic = dict(enable=True, filter_type=2)
    want = _frame(product, strict, city, stf=cubic)
    refused = [dict(enable=True, filter_type=4), dict(enable=True, filter_type=1, gaussian_sigma=0.0), dict(enable=True, filter_type=3, gaussian_sigma=-1.0),
               dict(enable=True, filter_type=3, gaussian_sigma=float("nan")), dict(enable=True, filter_type=3, gaussian_sigma=float("inf"))] + \
              [dict(enable=True, filter_type=1, magnification_method=m) for m in range(1, 7)] + [dict(enable=True, filter_type=1, magnification_method=7)]
    got = _frame(product, strict, city, stf=cubic, refused=refused)
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("filt", [0, 1, 2, 3])
def test_filters_deterministic_and_batch_invariant(product, city, strict, filt):
    """measured: each filter changes the textured frame against hardware trilinear, two runs agree bit for bit, and 1 or 4 sub-samples per launch give the same frame"""
    stf = dict(enable=True, filter_type=filt, gaussian_sigma=0.3)
    a = _frame(product, strict, city, spp=4, stf=stf, batch=4)
    b = _frame(product, strict, city, spp=4, stf=stf, batch=4)
    one = _frame(product, strict, city, spp=4, stf=stf, batch=1)
    assert a.tobytes() == b.tobytes() and a.tobytes() == one.tobytes()
    assert np.isfinite(a).all()
    base = _frame(product, strict, city, spp=4, batch=4)
    assert a.tobytes() != base.tobytes()
    # the same scene: STF changes the texels, not the image's brightness (4 spp, a loose bar on the mean)
    assert abs(a[..., :3].mean() / base[..., :3].mean() - 1) < 0.1


@pytest.mark.parametrize("strict", [False, True])
def test_realtime_passes(product, city, strict):
    """BUILD and FILL with STF: deterministic, and off again gives back a context that never enabled it"""
    from rtxpt_b200 import scene_builder as sb
    scene, cam, consts = city
    def run(first, second):
        """two frames, STF (cubic) on or off for each"""
        c = product.Context(max_sub_samples_per_launch=2, strict=strict)
        c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
        c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=3, sub_samples=2))
        c.set_texture_filtering(first, 2); c.path_trace_realtime(True); c.synchronize()
        c.set_texture_filtering(second, 2); c.path_trace_realtime(True); c.synchronize()
        r = c.readback_realtime(); c.close()
        return r
    base, on1, on2, back = run(False, False), run(True, True), run(True, True), run(True, False)
    for k in base:
        assert on1[k].tobytes() == on2[k].tobytes(), k
        assert back[k].tobytes() == base[k].tobytes(), k
    assert on1["merged"].tobytes() != base["merged"].tobytes()
    assert np.isfinite(on1["merged"]).all()
