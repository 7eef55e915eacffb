"""GPU: the CUDA ReBLUR chain (rtxpt_b200/csrc/reblur_kernels.cu; SURVEY §8 row a18 / K9) against the oracle's restatement (oracle/reblur.h), frame by frame through the
C ABI: realtime path trace -> rtxpt_b200_denoiser_prepare_inputs -> rtxpt_b200_reblur_denoise, with the oracle denoising the very inputs the product prepared, each side keeping
its own history.  Values are fp16 images; the two sides differ by libdevice vs glibc transcendentals (exp, pow, atan, log) in weights, so the bar is agreement within a few fp16
steps on nearly every pixel plus identical history-length bookkeeping, stated per assert.

Tolerances marked "measured" come from GPU runs of these tests."""
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


def _scene(product, strict, W, H):
    from rtxpt_b200 import scene_builder as sb, scenes
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    return c, cam, consts


def _moved(cam, W, H, dx):
    """The Cornell camera moved sideways by dx (same orientation)."""
    from rtxpt_b200 import scene_builder as sb
    out = type(cam).from_buffer_copy(bytes(cam))
    pos = np.array(cam.PosW[:], np.float32); right = np.array(cam.CameraU[:], np.float32); right /= np.linalg.norm(right)
    out.PosW[:] = (pos + right * dx).tolist()
    return out


def _frame(c, sb, W, H, cam, prev_cam, consts, frame_index, plane, reset=False):
    """One frame of the product: trace, prepare NRD's inputs of `plane`, denoise; returns (inputs, outputs)."""
    consts.sampleBaseIndex = frame_index
    c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=1, prev_cam=prev_cam))
    c.path_trace_realtime(False)
    c.denoiser_prepare_inputs(plane, True, sb.make_denoiser_constants(cam))
    c.reblur_denoise(plane, sb.make_reblur_frame(cam, prev_cam, frame_index=frame_index, reset=reset))
    c.synchronize()
    return c.readback_denoiser_inputs(), c.readback_reblur()


def _compare(out, od, os_, frames, inputs, min_close, label):
    surf = inputs["view_z"] < 1e5
    assert surf.mean() > 0.5
    for name, a, b in (("diff", out["diff"], od), ("spec", out["spec"], os_)):
        a = a.astype(np.float32)[surf]; b = b.astype(np.float32)[surf]
        assert np.isfinite(a).all(), (label, name)
        close = np.isclose(a, b, rtol=1e-2, atol=2e-3).all(-1).mean()
        assert close > min_close, (label, name, close)
        assert abs(a[..., 0].mean() - b[..., 0].mean()) < 0.01 * max(b[..., 0].mean(), 1e-3), (label, name)
    same_frames = (np.abs(out["frames"] - frames) < 0.3)[surf].all(-1).mean()                   # RG8 steps are 63 / 255 ~ 0.25 frames
    assert same_frames > min_close, (label, same_frames)


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_reblur_static_camera_matches_oracle(product, oracle, strict):
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    c, cam, consts = _scene(product, strict, W, H)
    rb = oracle.Reblur()
    wv, vc = sb.world_to_view(cam), sb.view_to_clip(cam)
    for f in range(5):
        inputs, out = _frame(c, sb, W, H, cam, cam, consts, f, plane=0)
        od, os_, frames = rb.denoise(wv, vc, f, inputs["view_z"], inputs["normal_roughness"], inputs["diff"], inputs["spec"], motion=inputs["motion"], disocclusion_mix=inputs["disocclusion_mix"])
        _compare(out, od, os_, frames, inputs, 0.985 if strict else 0.93, ("static", strict, f))
        surf = inputs["view_z"] < 1e5
        assert np.median(out["frames"][surf][:, 0]) >= min(f, 3) - 0.13                                 # history grows by one frame per frame on a static view
    rb.close(); c.close()


@unverified
def test_reblur_moving_camera_reprojects_like_the_oracle(product, oracle):
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    c, cam0, consts = _scene(product, True, W, H)
    rb = oracle.Reblur()
    prev = cam0
    for f in range(4):
        cam = _moved(cam0, W, H, 0.01 * f)
        inputs, out = _frame(c, sb, W, H, cam, prev, consts, f, plane=0)
        od, os_, frames = rb.denoise(sb.world_to_view(cam), sb.view_to_clip(cam), f, inputs["view_z"], inputs["normal_roughness"], inputs["diff"], inputs["spec"],
                                     prev_world_to_view=sb.world_to_view(prev), prev_view_to_clip=sb.view_to_clip(prev), motion=inputs["motion"], disocclusion_mix=inputs["disocclusion_mix"])
        _compare(out, od, os_, frames, inputs, 0.97, ("moving", f))
        prev = cam
    surf = inputs["view_z"] < 1e5
    assert np.median(out["frames"][surf][:, 0]) >= 2 - 0.13                                             # most of the diffuse history survived the motion
    rb.close(); c.close()


@unverified
def test_reblur_reset_and_per_plane_history(product):
    """History is per plane and a reset drops it: plane 1's first frame starts at 0 accumulated frames while plane 0 has history; a reset frame on plane 0 starts over."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    c, cam, consts = _scene(product, False, W, H)
    for f in range(3): inputs, out = _frame(c, sb, W, H, cam, cam, consts, f, plane=0)
    surf = inputs["view_z"] < 1e5
    assert np.median(out["frames"][surf][:, 0]) >= 2 - 0.13
    inputs1, out1 = _frame(c, sb, W, H, cam, cam, consts, 3, plane=1)
    s1 = inputs1["view_z"] < 1e5
    if s1.any(): assert out1["frames"][s1].max() == 0
    _, out2 = _frame(c, sb, W, H, cam, cam, consts, 4, plane=0, reset=True)
    assert out2["frames"][surf].max() == 0
    # replay determinism of a whole frame
    a = _frame(c, sb, W, H, cam, cam, consts, 5, plane=0, reset=True)[1]; b = _frame(c, sb, W, H, cam, cam, consts, 5, plane=0, reset=True)[1]
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)
    c.close()


@unverified
def test_denoise_realtime_reduces_error_and_keeps_energy(product):
    """Sample::Denoise end to end: the denoised frames converge towards the reference-mode image faster than the no-denoiser merge, without losing energy."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 160, 120
    c, cam, consts = _scene(product, False, W, H)
    consts.sampleBaseIndex = 0; c.set_constants(consts); c.reset_accumulation(); c.path_trace(0, 256, True); c.synchronize()
    ref = c.readback_accumulated()[..., :3].astype(np.float32)
    k = sb.make_denoiser_constants(cam)
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=1))
    for f in range(12):
        consts.sampleBaseIndex = 1000 + f; c.set_constants(consts)
        c.path_trace_realtime(True); c.synchronize(); noisy = c.readback_output_color()[..., :3].astype(np.float32)
        c.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=f)); c.synchronize(); den = c.readback_output_color()[..., :3].astype(np.float32)
    assert np.isfinite(den).all()
    e_noisy = np.abs(np.minimum(noisy, 4) - np.minimum(ref, 4)).mean(); e_den = np.abs(np.minimum(den, 4) - np.minimum(ref, 4)).mean()
    assert e_den < 0.6 * e_noisy, (e_den, e_noisy)                    # the 256 spp reference still carries noise of its own: the ratio understates the gain
    assert abs(den.mean() - ref.mean()) < 0.1 * ref.mean(), (den.mean(), ref.mean())
    c.close()


@unverified
def test_spec_hit_t_guide_filter_matches_oracle(product, oracle):
    """rtxpt_b200_denoise_spec_hit_t (DenoisingGuidesBaker::DenoiseSpecHitT) on the guide a realtime frame left behind: compare / add / divide only, so bit-identical."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    c, cam, consts = _scene(product, True, W, H)
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=1)); c.path_trace_realtime(False); c.synchronize()
    before = c.readback_realtime()
    c.denoise_spec_hit_t(); c.synchronize()
    after = c.readback_realtime()["spec_hit_t"]
    assert np.array_equal(after, oracle.denoise_spec_hit_t(before["depth"], before["spec_hit_t"]))
    c.close()
