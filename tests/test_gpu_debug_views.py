"""GPU: RTXPT's debug views (rtxpt_b200_set_debug_view) against the oracle's restatement (oracle/pt_debug_views.h, tests/oracle_debug_views_lib.py), both libraries.
  - first-hit views: the oracle loads the surface of each pixel's camera ray of the call's last sub-sample exactly as HandleHit does and colours it; the library draws the view
    from the surface its shade kernel loaded at vertex 1
  - stable-plane views: the oracle's StablePlanesDebugViz over the library's own plane buffers, so that the comparison is of the view and not of the paths
  - denoiser-merge views: the oracle's DENOISER_FINAL_MERGE debug switch over the library's own denoiser inputs and outputs, plane by plane
  - a view changes nothing else a call writes, DISABLED stops the writes, and refused views leave the context working."""
import numpy as np
import pytest

from rtxpt_b200 import structs as S

pytestmark = pytest.mark.gpu
V = S.DEBUG_VIEW
EXACT = (V["FirstHit_FrontFacing"], V["FirstHit_ThinSurface"], V["FirstHit_MaterialID"], V["FirstHit_ShaderID"])
GEOMETRY = (V["FirstHit_Barycentrics"], V["FirstHit_FaceNormal"], V["FirstHit_GeometryNormal"]) + EXACT
SPP = 5          # three launches of at most two sub-samples: only the call's last sub-sample draws


@pytest.fixture(scope="module")
def odv():
    import oracle_debug_views_lib
    oracle_debug_views_lib.build()
    return oracle_debug_views_lib


def _first_hit_views(product, odv, scene, consts, strict, views):
    c = product.Context(max_sub_samples_per_launch=2, strict=strict); c.upload_scene(scene); c.set_constants(consts)
    o = odv.oracle.Oracle(scene); o.set_constants(consts)
    out = {}
    for v in views:
        c.set_debug_view(v); c.reset_accumulation(); c.path_trace(0, SPP, True); c.synchronize()
        out[v] = (c.readback_debug_view(), odv.first_hit(o, v, consts.sampleBaseIndex + SPP - 1).astype(np.float16))
    c.close(); o.close()
    return out


@pytest.mark.parametrize("strict", [False, True])
def test_first_hit_views_cornell(product, odv, strict):
    """untextured Cornell box, all 14 views: strict build bit-identical on every pixel; default build within 1e-3, the flag and ID views exact"""
    from rtxpt_b200 import scenes, scene_builder as sb
    W = H = 128
    scene, cam = scenes.cornell_box(W, H)
    consts = sb.make_constants(W, H, cam, bounce_count=4, diffuse_bounce_count=3)
    for v, (img, ref) in _first_hit_views(product, odv, scene, consts, strict, S.DEBUG_VIEWS_FIRST_HIT).items():
        name = S.DEBUG_VIEW_NAMES[v]
        assert (ref[..., 3] == 1).mean() > 0.5, name                                  # most camera rays hit the room
        if strict or v in EXACT: assert np.array_equal(img.view(np.uint16), ref.view(np.uint16)), (name, int((img != ref).any(-1).sum()))
        else: assert np.abs(img.astype(np.float32) - ref.astype(np.float32)).max() <= 1e-3, name


def test_first_hit_views_textured_city(product, odv):
    """textured small city, strict build: the geometry views bit-identical on >= 99.9 % of the pixels (the two traversals may pick a different triangle where two meet);
    the texture-dependent views - hardware trilinear filtering against the oracle's - within 0.02 on >= 99 % of the pixels.  Observed on an H100: every geometry view and
    Specular, Metallic bit-identical on 100 % of the pixels; Diffuse on 3.5 % and Roughness on 94.5 % (the texture unit's 8-bit filter weights); every view within 0.02 on 100 %"""
    from rtxpt_b200 import scenes, scene_builder as sb
    W, H = 320, 180
    scene, cam = scenes.city_block(target_triangles=60000, width=W, height=H)
    consts = sb.make_constants(W, H, cam, bounce_count=4, diffuse_bounce_count=3, env_enabled=True)
    for v, (img, ref) in _first_hit_views(product, odv, scene, consts, True, S.DEBUG_VIEWS_FIRST_HIT).items():
        name = S.DEBUG_VIEW_NAMES[v]
        same = (img.view(np.uint16) == ref.view(np.uint16)).all(-1).mean()
        close = (np.abs(img.astype(np.float32) - ref.astype(np.float32)) <= 0.02).all(-1).mean()
        print(f"{name}: bit-identical {same:.5f}, within 0.02 {close:.5f}")
        if v in GEOMETRY: assert same >= 0.999, (name, same)
        else: assert close >= 0.99, (name, close)


def _realtime(product, strict, W=96, H=96):
    from rtxpt_b200 import scenes, scene_builder as sb
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=2)
    c.set_realtime(rt)
    return c, scene, consts, rt


def test_stable_plane_views(product, odv):
    """realtime Cornell box with delta surfaces, strict build: every StablePlanesDebugViz view at planes 0-2 and the four-way split is the oracle's over the same buffers"""
    c, scene, consts, rt = _realtime(product, True)
    o = odv.oracle.Oracle(scene); o.set_constants(consts)
    for v in S.DEBUG_VIEWS_STABLE_PLANES:
        for plane in (0, 1, 2, -1):
            c.set_debug_view(v, plane); c.path_trace_realtime(True); c.synchronize()
            img = c.readback_debug_view(); buffers = c.readback_realtime()
            ref = odv.stable_planes(o, rt, v, plane, buffers).astype(np.float16)
            assert np.array_equal(img.view(np.uint16), ref.view(np.uint16)), (S.DEBUG_VIEW_NAMES[v], plane, int((img != ref).any(-1).sum()))
    # the first-hit views in realtime mode come from the BUILD pass, whose camera ray is the reference mode's of sample index sampleBaseIndex
    for v in (V["FirstHit_ShadingNormal"], V["FirstHit_MaterialID"]):
        c.set_debug_view(v); c.path_trace_realtime(True); c.synchronize()
        ref = odv.first_hit(o, v, consts.sampleBaseIndex).astype(np.float16)
        assert np.array_equal(c.readback_debug_view().view(np.uint16), ref.view(np.uint16)), S.DEBUG_VIEW_NAMES[v]
    c.close(); o.close()


def _merge_pair(c, odv, o, rt, k, view, plane_index, viz):
    """one merge per plane, last to first, with the prepared inputs as the denoised images (identity denoiser); the oracle draws from the library's own targets after each"""
    for plane in range(rt.activeStablePlaneCount - 1, -1, -1):
        c.denoiser_prepare_inputs(plane, plane == rt.activeStablePlaneCount - 1, k); c.denoiser_final_merge(plane); c.synchronize()
        realtime = c.readback_realtime(); den = c.readback_denoiser_inputs(); den["output"] = c.readback_output_color()
        odv.denoiser_merge(o, rt, plane, plane_index, view, realtime, den, den["diff"], den["spec"], viz)


def test_denoiser_merge_views(product, odv):
    """realtime Cornell box with delta surfaces, strict build: every DENOISER_FINAL_MERGE view at planes 0-2 and the four-way split is the oracle's over the same inputs,
    through rtxpt_b200_denoiser_final_merge plane by plane and through rtxpt_b200_denoise_realtime (ReBLUR's outputs as the denoised images)"""
    from rtxpt_b200 import scene_builder as sb
    c, scene, consts, rt = _realtime(product, True)
    from rtxpt_b200 import scenes
    _, cam = scenes.cornell_box(96, 96, delta_surfaces=True)
    k = sb.make_denoiser_constants(cam)
    o = odv.oracle.Oracle(scene); o.set_constants(consts)
    for v in S.DEBUG_VIEWS_DENOISER_MERGE:
        for plane in (0, 1, 2, -1):
            c.set_debug_view(v, plane); c.path_trace_realtime(False)
            viz = np.zeros((96, 96, 4), np.float32)
            _merge_pair(c, odv, o, rt, k, v, plane, viz)
            with np.errstate(over="ignore"): ref = viz.astype(np.float16)       # ViewZ of a sky pixel: FLT_MAX / 10, infinite in fp16 as on the GPU
            img = c.readback_debug_view()
            assert np.array_equal(img.view(np.uint16), ref.view(np.uint16)), (S.DEBUG_VIEW_NAMES[v], plane, int((img.view(np.uint16) != ref.view(np.uint16)).any(-1).sum()))
            assert (ref[..., 3] == 1).mean() > (0.2 if plane == -1 and v != V["StablePlane_DenoiserValidation"] else 0.99)
        c.set_debug_view(v, 0); c.path_trace_realtime(False); c.denoise_realtime(k, sb.make_reblur_frame(cam, cam)); c.synchronize()
        realtime = c.readback_realtime(); den = c.readback_denoiser_inputs(); den["output"] = c.readback_output_color(); rb = c.readback_reblur()
        viz = np.zeros((96, 96, 4), np.float32)
        odv.denoiser_merge(o, rt, 0, 0, v, realtime, den, rb["diff"], rb["spec"], viz)
        with np.errstate(over="ignore"): ref = viz.astype(np.float16)
        assert np.array_equal(c.readback_debug_view().view(np.uint16), ref.view(np.uint16)), S.DEBUG_VIEW_NAMES[v]
    c.close(); o.close()


def test_one_active_plane_shows_plane_0(product, odv):
    """with one active stable plane every plane index shows plane 0 (Sample.cpp:2161)"""
    from rtxpt_b200 import scenes, scene_builder as sb
    W = H = 64
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=True); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, active_planes=1, bounce_count=8, sub_samples=1); c.set_realtime(rt)
    o = odv.oracle.Oracle(scene); o.set_constants(consts)
    for plane in (2, S.DEBUG_VIEW_STABLE_PLANE_SPLIT):
        c.set_debug_view(V["StablePlane_Normals"], plane); c.path_trace_realtime(True); c.synchronize()
        ref = odv.stable_planes(o, rt, V["StablePlane_Normals"], 0, c.readback_realtime()).astype(np.float16)
        assert np.array_equal(c.readback_debug_view().view(np.uint16), ref.view(np.uint16)), plane
    c.close(); o.close()


def _same(a, b):
    return all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


VARIANTS = {"stf": dict(), "nee_full_samples": dict(nee_full=3), "approximate_mis": dict(approximate_mis=True), "stf_nee_full_samples_approximate_mis": dict(nee_full=2, approximate_mis=True)}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_debug_kernel_variants_change_nothing_else(product, odv, variant):
    """the first-hit debug kernels of stochastic texture filtering, NEEFullSamples > 1 and approximate MIS: accumulation, output and guides bit-identical to the same call
    without the view, in both builds and with and without guides; the view is the oracle's"""
    from rtxpt_b200 import scenes, scene_builder as sb
    W = H = 64
    scene, cam = scenes.cornell_box(W, H)
    consts = sb.make_constants(W, H, cam, bounce_count=4, diffuse_bounce_count=3, **VARIANTS[variant])
    o = odv.oracle.Oracle(scene); o.set_constants(consts)
    ref = odv.first_hit(o, V["FirstHit_ShadingNormal"], consts.sampleBaseIndex + 3).astype(np.float16)
    for strict in (False, True):
        for flags in (0, S.CFG_EXPORT_GUIDES):
            c = product.Context(max_sub_samples_per_launch=2, strict=strict, flags=flags); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
            if variant.startswith("stf"): c.set_texture_filtering(True, S.STF_FILTER_LINEAR, 0, 0.3)

            def frame():
                c.reset_accumulation(); c.path_trace(0, 4, True); c.synchronize()
                return [c.readback_accumulated(), c.readback_output_color()] + (list(c.readback_guides()) if flags else [])

            base = frame(); c.set_debug_view(V["FirstHit_ShadingNormal"])
            assert _same(base, frame()), (strict, flags)
            img = c.readback_debug_view()
            if strict: assert np.array_equal(img.view(np.uint16), ref.view(np.uint16)), (strict, flags)
            else: assert np.abs(img.astype(np.float32) - ref.astype(np.float32)).max() <= 1e-3, (strict, flags)
            c.close()
    o.close()


@pytest.mark.parametrize("strict", [False, True])
def test_views_change_nothing_else(product, strict):
    """a view leaves every other target of both modes bit-identical; DISABLED stops the writes; a refused view returns RTXPT_ERR_UNSUPPORTED and the context renders on"""
    from rtxpt_b200 import lib, scenes, scene_builder as sb
    W = H = 96
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=2, strict=strict, flags=S.CFG_EXPORT_GUIDES); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))

    def reference():
        c.reset_accumulation(); c.path_trace(0, 4, True); c.synchronize()
        return [c.readback_accumulated(), c.readback_output_color()] + list(c.readback_guides())

    base = reference()
    for v in (V["FirstHit_ShadingNormal"], V["FirstHit_Diffuse"], V["StablePlane_Normals"]):
        c.set_debug_view(v)
        assert _same(base, reference()), S.DEBUG_VIEW_NAMES[v]
    c.set_debug_view(V["FirstHit_ShadingNormal"]); reference(); drawn = c.readback_debug_view()
    assert (drawn[..., 3] == 1).mean() > 0.5
    c.set_debug_view(V["Disabled"]); reference()
    assert np.array_equal(c.readback_debug_view(), drawn)                        # nothing cleared or drawn once disabled

    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2); c.set_realtime(rt)

    def realtime():
        c.path_trace_realtime(True); c.synchronize()
        return [c.readback_output_color()] + list(c.readback_realtime().values())

    base_rt = realtime()
    for v in (V["FirstHit_ShadingNormal"], V["DominantStablePlaneIndex"], V["StableRadiance"]):
        c.set_debug_view(v)
        assert _same(base_rt, realtime()), S.DEBUG_VIEW_NAMES[v]
    k = sb.make_denoiser_constants(cam)

    def denoised():     # the merge of every plane with the prepared inputs as the denoised images (ReBLUR's history would move between the calls)
        c.path_trace_realtime(False)
        for plane in (2, 1, 0): c.denoiser_prepare_inputs(plane, plane == 2, k); c.denoiser_final_merge(plane)
        c.synchronize()
        return [c.readback_output_color()] + list(c.readback_denoiser_inputs().values())

    c.set_debug_view(V["Disabled"]); base_dn = denoised()
    for v in (V["StablePlane_ViewZ"], V["StablePlane_CombinedRadianceDenoised"]):
        c.set_debug_view(v, S.DEBUG_VIEW_STABLE_PLANE_SPLIT)
        assert _same(base_dn, denoised()), S.DEBUG_VIEW_NAMES[v]

    c.set_debug_view(V["StablePlane_Roughness"], 1)
    for v in (V["DenoiserGuide_Depth"], V["DenoiserGuide_PrimaryLayer"], V["VBufferMotionVectors"], V["ReSTIRDIFinalOutput"]):
        with pytest.raises(lib.RtxptError, match="error -6"): c.set_debug_view(v)
    with pytest.raises(lib.RtxptError, match="error -1"): c.set_debug_view(S.DEBUG_VIEW_MAX_COUNT)
    with pytest.raises(lib.RtxptError, match="error -1"): c.set_debug_view(V["StablePlane_Normals"], 3)
    assert _same(base_rt, realtime())
    kept = c.readback_debug_view()                                                 # the view set before the refusals is still drawn
    c.set_debug_view(V["StablePlane_Roughness"], 1); realtime()
    assert np.array_equal(c.readback_debug_view(), kept)
    c.close()
