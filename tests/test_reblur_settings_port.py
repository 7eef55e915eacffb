"""CPU: ReBLUR under the settings RTXPT's denoiser panel sets (RtxptReblurSettings, rtxpt_b200_set_reblur_settings), the CUDA source held to the oracle without a GPU.
The host build of the product's passes under settings (tests/emu/reblur_settings_host_emu.cu: reblur_passes.cuh, the validation, host constants and pass routing of reblur_host.h)
and the oracle's (oracle/reblur_settings.h, which restates NRD's dispatch graph for the settings on reblur.h's passes) must agree bit for bit for every reconstruction mode (OFF / 3x3 / 5x5), for pre-pass radii that skip the pre-pass or one of its
halves, with anti-firefly and the disocclusion-threshold mix off, and with every numeric field away from its default.  The validation mirror (structs.reblur_settings_status) is
held to the product's own check."""
import numpy as np
import pytest
import reblur_inputs as ri
import reblur_settings_lib as rsl
from test_reblur_port import _both, _assert_identical

W, H = 80, 64


def _settings(**changes):
    from rtxpt_b200 import structs as S
    return S.ReblurSettings.default(**changes)


# RTXPT's defaults are 5x5 reconstruction, pre-pass radii (15, 40), anti-firefly and the mix on
CASES = {
    "off": dict(hitDistanceReconstructionMode=0),
    "3x3": dict(hitDistanceReconstructionMode=1),
    "5x5": dict(),
    "prepass_0_0": dict(diffusePrepassBlurRadius=0.0, specularPrepassBlurRadius=0.0),
    "prepass_0_40": dict(diffusePrepassBlurRadius=0.0, specularPrepassBlurRadius=40.0),
    "prepass_15_0": dict(diffusePrepassBlurRadius=15.0, specularPrepassBlurRadius=0.0),
    "off_prepass_0_0": dict(hitDistanceReconstructionMode=0, diffusePrepassBlurRadius=0.0, specularPrepassBlurRadius=0.0),
    "3x3_prepass_0_0": dict(hitDistanceReconstructionMode=1, diffusePrepassBlurRadius=0.0, specularPrepassBlurRadius=0.0),
    "off_prepass_15_0": dict(hitDistanceReconstructionMode=0, diffusePrepassBlurRadius=15.0, specularPrepassBlurRadius=0.0),
    "antifirefly_off": dict(enableAntiFirefly=0),
    "mix_off": dict(useAlternateDisocclusionThresholdMix=0),
    "all_changed": dict(hitDistanceParameters=(2.5, 0.15, 12.0, -18.0), antilagLuminanceSigmaScale=2.0, antilagLuminanceSensitivity=1.5, maxAccumulatedFrameNum=24,
                        maxFastAccumulatedFrameNum=4, historyFixFrameNum=0, diffusePrepassBlurRadius=9.0, specularPrepassBlurRadius=22.0, minBlurRadius=2.0, maxBlurRadius=18.0,
                        lobeAngleFraction=0.3, roughnessFraction=0.25, responsiveAccumulationRoughnessThreshold=0.35, planeDistanceSensitivity=0.05, hitDistanceReconstructionMode=1,
                        enableAntiFirefly=0, useAlternateDisocclusionThresholdMix=0),
}


_rendered = {}


def _rendered_frame(oracle, plane, key, cam, prev, index):
    """The oracle's realtime render of the Cornell box (delta surfaces, so that plane 1 exists) for one camera, kept for every settings case."""
    from rtxpt_b200 import scene_builder as sb, scenes
    if "oracle" not in _rendered:
        scene, _ = scenes.cornell_box(W, H, delta_surfaces=True); _rendered["oracle"] = oracle.Oracle(scene)
    o = _rendered["oracle"]
    if key not in _rendered:
        c = sb.make_constants(W, H, cam, bounce_count=4, diffuse_bounce_count=3); c.sampleBaseIndex = index
        o.set_constants(c); o.set_view(sb.world_to_clip(cam))
        rt = sb.make_realtime_constants(W, H, cam, prev_cam=prev, bounce_count=4, sub_samples=1)
        _rendered[key] = (rt, o.render_realtime(rt))
    return o, _rendered[key]


def dolly_inputs(oracle, plane, hit_params):
    """NRD inputs of one plane along the sequence of test_reblur_port's dolly: five frames of a slow dolly, an undescribed cut (no motion vectors), a reset.  Yields
    (camera, previous camera, frame index, inputs, reset, use motion vectors); the inputs are normalised with `hit_params` (RtxptDenoiserConstants::hitDistanceParameters)."""
    from rtxpt_b200 import scene_builder as sb
    cam_at = lambda dx: sb.bridge_camera(W, H, pos=(2.78 + dx, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    cut = sb.bridge_camera(W, H, pos=(4.2, 1.2, -6.0), direction=(-0.25, 0.1, 1), up=(0, 1, 0), fov_y=0.66)
    seq = [(cam_at(0.03 * f), cam_at(0.03 * (f - 1)) if f else None, f, f, False, True) for f in range(5)] + [(cut, cut, 20, 5, False, False), (cut, cut, 21, 6, True, True)]
    for cam, prev, render_index, f, reset, motion in seq:
        o, (rt, r) = _rendered_frame(oracle, plane, ("frame", render_index), cam, prev, render_index)
        d = o.new_denoiser_targets()
        o.denoiser_prepare_inputs(rt, sb.make_denoiser_constants(cam, hit_distance_parameters=hit_params), r, d, plane, True)
        yield cam, prev, f, d, reset, motion


@pytest.mark.parametrize("plane", [0, 1])
@pytest.mark.parametrize("case", sorted(CASES))
def test_port_equals_oracle_on_a_dolly_with_settings(oracle, case, plane):
    """Every case along the dolly, the cut and the reset, bit for bit; the settings are set once before the first frame."""
    from rtxpt_b200 import scene_builder as sb
    s = _settings(**CASES[case])
    rb = rsl.OracleReblur(); port = rsl.PortReblur()
    rb.set(s); assert port.set(s) == 0
    grown = 0.0
    for cam, prev, f, d, reset, motion in dolly_inputs(oracle, plane, tuple(s.hitDistanceParameters)):
        a, b = _both(rb, port, sb, cam, prev, f, d, reset=reset, use_motion=motion)
        surf = d["view_z"] < 1e30
        _assert_identical(a, b, surf, (case, plane, f))
        if surf.any() and not reset: grown = max(grown, float(b[2][surf].max()))
    assert grown >= 3 or s.maxAccumulatedFrameNum < 3                                       # the history grew, so the temporal paths ran
    assert (b[2] == 0).all()                                                                 # the reset frame
    rb.close(); port.close()


def test_settings_change_mid_sequence_keeps_history(oracle):
    """Settings changed between frames (5x5 -> OFF without pre-pass -> 3x3 with anti-firefly off) take effect on the next frame and keep the history, as in NRD; port and oracle agree."""
    from rtxpt_b200 import scene_builder as sb
    rb = rsl.OracleReblur(); port = rsl.PortReblur()
    changes = {2: _settings(**CASES["off_prepass_0_0"]), 4: _settings(hitDistanceReconstructionMode=1, enableAntiFirefly=0)}
    for cam, prev, f, d, reset, motion in dolly_inputs(oracle, 0, (3.0, 0.1, 20.0, -25.0)):
        if f in changes: rb.set(changes[f]); assert port.set(changes[f]) == 0
        a, b = _both(rb, port, sb, cam, prev, f, d, reset=reset, use_motion=motion)
        surf = d["view_z"] < 1e30
        _assert_identical(a, b, surf, ("change", f))
        if f == 2: assert b[2][surf].max() >= 2 - 0.13                                      # the history survived the change (RG8 steps of 63 / 255)
    rb.close(); port.close()


def test_default_settings_reproduce_the_unset_denoiser(oracle):
    """The oracle's and the port's instances with settings, given rtxpt_b200_default_reblur_settings' values, denoise exactly as the committed oracle (oracle.Reblur) and the
    committed host build (host_build_lib.ReblurPort), which know no settings: RTXPT's configuration is unchanged."""
    from rtxpt_b200 import scene_builder as sb
    import host_build_lib as emu
    rb0, rb1, p0, p1 = oracle.Reblur(), rsl.OracleReblur(), emu.ReblurPort(), rsl.PortReblur()
    s = _settings(); rb1.set(s); assert p1.set(s) == 0
    for cam, prev, f, d, reset, motion in dolly_inputs(oracle, 1, (3.0, 0.1, 20.0, -25.0)):
        a0, b0 = _both(rb0, p0, sb, cam, prev, f, d, reset=reset, use_motion=motion)
        a1, b1 = _both(rb1, p1, sb, cam, prev, f, d, reset=reset, use_motion=motion)
        everywhere = np.ones(d["view_z"].shape, bool)
        _assert_identical(a0, a1, everywhere, ("oracle default", f)); _assert_identical(b0, b1, everywhere, ("port default", f))
    for x in (rb0, rb1, p0, p1): x.close()


@pytest.mark.parametrize("W_,H_", ri.SHAPES)
def test_3x3_port_equals_oracle_at_tile_and_image_edges(oracle, W_, H_):
    """The 3x3 reconstruction on tests/reblur_inputs.py's synthetic frames (sky tiles, zero hit distances on seams and borders) at frame sizes with partial tiles, no interior tile,
    one tile and one column: a reset, two static frames, two moving ones; every pixel, sky included."""
    from rtxpt_b200 import scene_builder as sb
    rb = rsl.OracleReblur(); port = rsl.PortReblur(); s = _settings(hitDistanceReconstructionMode=1)
    rb.set(s); assert port.set(s) == 0
    cam = prev = ri.camera(W_, H_)
    everywhere = np.ones((H_, W_), bool)
    for f in range(3):
        a, b = _both(rb, port, sb, cam, cam, f, ri.inputs(W_, H_, frame=f), reset=f == 0)
        _assert_identical(a, b, everywhere, (W_, H_, f))
    for f in range(3, 5):
        cam = ri.moved_camera(W_, H_, f - 2)
        a, b = _both(rb, port, sb, cam, prev, f, ri.inputs(W_, H_, frame=f, motion=(-1.3, 0.6)))
        _assert_identical(a, b, everywhere, (W_, H_, "moving", f))
        prev = cam
    rb.close(); port.close()


def validation_cases():
    """(label, settings) pairs on both sides of every bound the setter checks"""
    nan, inf = float("nan"), float("inf")
    out = [("default", {})]
    for k in ("antilagLuminanceSigmaScale", "antilagLuminanceSensitivity", "diffusePrepassBlurRadius", "specularPrepassBlurRadius", "minBlurRadius", "maxBlurRadius",
              "lobeAngleFraction", "roughnessFraction", "responsiveAccumulationRoughnessThreshold", "planeDistanceSensitivity"):
        out += [(k + " nan", {k: nan}), (k + " inf", {k: inf}), (k + " -inf", {k: -inf}), (k + " 0", {k: 0.0}), (k + " -0.001", {k: -0.001}), (k + " 1", {k: 1.0}),
                (k + " 1.001", {k: 1.001}), (k + " 250", {k: 250.0})]
    for i in range(4):
        for v in (nan, inf, -inf, -7.0, 0.0, 1e6):
            hp = [3.0, 0.1, 20.0, -25.0]; hp[i] = v; out.append(("hit %d %g" % (i, v), {"hitDistanceParameters": hp}))
    for k in ("maxAccumulatedFrameNum", "maxFastAccumulatedFrameNum", "historyFixFrameNum"):
        out += [(k + " %d" % v, {k: v}) for v in (0, 1, 62, 63, 64, 1000, 0xFFFFFFFF)]
    out += [("mode %d" % v, {"hitDistanceReconstructionMode": v}) for v in (0, 1, 2, 3, 255)]
    for k in ("enableAntiFirefly", "useAlternateDisocclusionThresholdMix"):
        out += [(k + " %d" % v, {k: v}) for v in (0, 1, 2, 0xFFFFFFFF)]
    out.append(("all_changed", CASES["all_changed"]))
    return out


def test_validation_mirror_refuses_what_the_product_refuses(oracle):
    """structs.reblur_settings_status against the product's check (reblur_host.h settingsError, the one rtxpt_b200_set_reblur_settings runs), and a refused call keeps the
    previous settings: the instance keeps denoising with what it had."""
    from rtxpt_b200 import structs as S, scene_builder as sb
    port = rsl.PortReblur()
    refused = 0
    for label, ch in validation_cases():
        s = _settings(**ch)
        want = S.reblur_settings_status(s)
        assert port.set(s) == want, label
        refused += want != 0
    assert refused > 60
    # a refused call after an accepted one: the accepted settings stay
    rb = rsl.OracleReblur(); p2 = rsl.PortReblur(); good = _settings(**CASES["3x3_prepass_0_0"])
    rb.set(good); assert p2.set(good) == 0
    assert p2.set(_settings(hitDistanceReconstructionMode=3, diffusePrepassBlurRadius=15.0)) == -1
    for cam, prev, f, d, reset, motion in list(dolly_inputs(oracle, 0, (3.0, 0.1, 20.0, -25.0)))[:3]:
        a, b = _both(rb, p2, sb, cam, prev, f, d, reset=reset, use_motion=motion)
        _assert_identical(a, b, d["view_z"] < 1e30, ("kept", f))
    for x in (port, rb, p2): x.close()
