"""GPU: ReBLUR under the settings RTXPT's denoiser panel sets (rtxpt_b200_set_reblur_settings), both libraries.

Every settings case of tests/test_reblur_settings_port.py against the oracle on realtime Cornell frames, at the bars of tests/test_gpu_reblur.py; the 3x3 reconstruction at the frame
shapes of tests/test_gpu_reblur_shapes.py (tiled equals untiled bit for bit, including 1080p; per-band bars against the oracle); the default settings give frames bit-identical to a
context that never called the setter; a refused call changes nothing; a whole denoise_realtime frame with non-default settings against the oracle's ReBLUR; two contexts of a tile
group denoise identically after the setter."""
import ctypes as C
import numpy as np
import pytest
import reblur_inputs as ri
from test_gpu_reblur import _scene, _moved, _compare
from test_gpu_reblur_shapes import _context, _frames as _shape_frames, _denoise, _compare_with_oracle
import reblur_settings_lib as rsl
from test_reblur_settings_port import CASES, _settings, validation_cases

HIT = (3.0, 0.1, 20.0, -25.0)


def _frame(c, sb, W, H, cam, prev_cam, consts, frame_index, plane, hit_params, reset=False):
    consts.sampleBaseIndex = frame_index
    c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=1, prev_cam=prev_cam))
    c.path_trace_realtime(False)
    c.denoiser_prepare_inputs(plane, True, sb.make_denoiser_constants(cam, hit_distance_parameters=hit_params))
    c.reblur_denoise(plane, sb.make_reblur_frame(cam, prev_cam, frame_index=frame_index, reset=reset))
    c.synchronize()
    return c.readback_denoiser_inputs(), c.readback_reblur()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("case", sorted(CASES))
def test_settings_match_oracle(product, strict, case):
    """Four static frames (the bars of test_reblur_static_camera_matches_oracle), then, in the strict build, three frames of a moving camera (the bar of
    test_reblur_moving_camera_reprojects_like_the_oracle); the oracle denoises the inputs the product prepared, with the same settings."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    s = _settings(**CASES[case]); hp = tuple(s.hitDistanceParameters)
    c, cam0, consts = _scene(product, strict, W, H)
    c.set_reblur_settings(s)
    rb = rsl.OracleReblur(); rb.set(s)
    seq = [(cam0, cam0, f, 0.985 if strict else 0.93) for f in range(4)]
    if strict: seq += [(_moved(cam0, W, H, 0.01 * f), _moved(cam0, W, H, 0.01 * (f - 1)), 3 + f, 0.97) for f in range(1, 4)]
    for cam, prev, f, bar in seq:
        inputs, out = _frame(c, sb, W, H, cam, prev, consts, f, 0, hp)
        od, os_, frames = rb.denoise(sb.world_to_view(cam), sb.view_to_clip(cam), f, inputs["view_z"], inputs["normal_roughness"], inputs["diff"], inputs["spec"],
                                     prev_world_to_view=sb.world_to_view(prev), prev_view_to_clip=sb.view_to_clip(prev), motion=inputs["motion"], disocclusion_mix=inputs["disocclusion_mix"])
        _compare(out, od, os_, frames, inputs, bar, (case, strict, f))
    rb.close(); c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("W,H", ri.SHAPES + [(1920, 1080)])
def test_3x3_tiled_equals_untiled(product, strict, W, H):
    """The 3x3 reconstruction through the shared-memory tile (24 x 18: TMA or clamped loads) and through global-memory taps: the same frames bit for bit, every pixel."""
    from rtxpt_b200 import structs as S
    s = _settings(hitDistanceReconstructionMode=1)
    tiled, untiled = _context(product, strict, W, H), _context(product, strict, W, H, flags=S.CFG_REBLUR_UNTILED)
    tiled.set_reblur_settings(s); untiled.set_reblur_settings(s)
    for d, cam, prev, f, reset in _shape_frames(W, H, moving=(W, H) == (100, 72)):
        a, b = _denoise(tiled, d, cam, prev, f, reset), _denoise(untiled, d, cam, prev, f, reset)
        for k in ("diff", "spec", "frames"):
            same = (a[k] == b[k]) | (np.isnan(a[k]) & np.isnan(b[k]))
            assert same.all(), (W, H, strict, f, k, int((~same.all(-1)).sum()))
    tiled.close(); untiled.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
@pytest.mark.parametrize("W,H", ri.SHAPES)
def test_3x3_matches_oracle_per_band(product, strict, W, H):
    """The 3x3 reconstruction against the oracle on the synthetic frames, the per-band bars of test_gpu_reblur_shapes.py; frame counters and sky bit for bit."""
    from rtxpt_b200 import scene_builder as sb
    s = _settings(hitDistanceReconstructionMode=1)
    c = _context(product, strict, W, H); c.set_reblur_settings(s)
    rb = rsl.OracleReblur(); rb.set(s)
    for d, cam, prev, f, reset in _shape_frames(W, H, moving=False):
        out = _denoise(c, d, cam, prev, f, reset)
        od, os_, frames = rb.denoise(sb.world_to_view(cam), sb.view_to_clip(cam), f, d["view_z"], d["normal_roughness"], d["diff"], d["spec"], prev_world_to_view=sb.world_to_view(prev),
                                     prev_view_to_clip=sb.view_to_clip(prev), motion=d["motion"], disocclusion_mix=d["disocclusion_mix"], reset=reset)
        _compare_with_oracle(out, od, os_, frames, d, strict, (W, H, strict, f))
    rb.close(); c.close()


def _sequence(c, sb, W, H, cam, consts, frames, hp=HIT):
    outs = []
    for f in range(frames):
        _, out = _frame(c, sb, W, H, cam, cam, consts, f, 0, hp)
        outs.append(out)
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
def test_default_settings_equal_a_context_that_never_set_them(product, strict):
    """rtxpt_b200_default_reblur_settings' values, set explicitly, give frames bit-identical to those of a context that never called the setter; the library's defaults are the
    Python mirror's."""
    from rtxpt_b200 import scene_builder as sb, structs as S
    W, H = 96, 80
    a, cam, consts = _scene(product, strict, W, H); b, _, _ = _scene(product, strict, W, H)
    d = S.ReblurSettings(); L = a.L; L.rtxpt_b200_default_reblur_settings(C.byref(d))
    assert bytes(d) == bytes(_settings())
    b.set_reblur_settings(d)
    for x, y in zip(_sequence(a, sb, W, H, cam, consts, 4), _sequence(b, sb, W, H, cam, consts, 4)):
        assert all(x[k].tobytes() == y[k].tobytes() for k in x)
    a.close(); b.close()


@pytest.mark.gpu
def test_refused_settings_change_nothing(product):
    """rtxpt_b200_set_reblur_settings refuses exactly what structs.reblur_settings_status refuses, and a refused call leaves the settings in force: a context that was refused
    settings between frames denoises bit for bit like one that was not."""
    from rtxpt_b200 import scene_builder as sb, structs as S, lib
    W, H = 96, 80
    a, cam, consts = _scene(product, False, W, H); b, _, _ = _scene(product, False, W, H)
    probe = product.Context(max_sub_samples_per_launch=1)
    for label, ch in validation_cases():
        s = _settings(**ch)
        if S.reblur_settings_status(s) == 0: probe.set_reblur_settings(s)
        else:
            with pytest.raises(lib.RtxptError): probe.set_reblur_settings(s)
    probe.close()
    good = _settings(**CASES["3x3_prepass_0_0"])
    a.set_reblur_settings(good); b.set_reblur_settings(good)
    for label, ch in validation_cases():
        s = _settings(**ch)
        if S.reblur_settings_status(s) != 0:
            with pytest.raises(lib.RtxptError): a.set_reblur_settings(s)
    for x, y in zip(_sequence(a, sb, W, H, cam, consts, 3), _sequence(b, sb, W, H, cam, consts, 3)):
        assert all(x[k].tobytes() == y[k].tobytes() for k in x)
    a.close(); b.close()


def _device_image(array):
    import torch
    return torch.from_numpy(np.ascontiguousarray(array).view(np.uint16).copy()).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
def test_denoise_realtime_frame_with_settings_matches_oracle(product, strict):
    """Sample::Denoise with non-default settings (every field changed, hit parameters in both places): one context runs rtxpt_b200_denoise_realtime; a twin context traces the
    same frames and runs the same chain pass by pass, with each plane's ReBLUR done by an oracle instance (one per plane) on the inputs it prepared and merged back by the
    library.  The two output colours agree within the bars of test_gpu_reblur.py's static frames."""
    import torch
    from rtxpt_b200 import scene_builder as sb
    W, H = 96, 80
    s = _settings(**CASES["all_changed"]); hp = tuple(s.hitDistanceParameters)
    a, cam, consts = _scene(product, strict, W, H); b, _, _ = _scene(product, strict, W, H)
    a.set_reblur_settings(s)
    rbs = [rsl.OracleReblur() for _ in range(3)]
    for rb in rbs: rb.set(s)
    k = sb.make_denoiser_constants(cam, hit_distance_parameters=hp)
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=1)
    for f in range(4):
        consts.sampleBaseIndex = f; frame = sb.make_reblur_frame(cam, cam, frame_index=f)
        for c in (a, b): c.set_constants(consts); c.set_realtime(rt); c.path_trace_realtime(False)
        a.denoise_realtime(k, frame); a.synchronize()
        b.denoise_spec_hit_t()
        for i, plane in enumerate((2, 1, 0)):
            b.denoiser_prepare_inputs(plane, i == 0, k); b.synchronize(); d = b.readback_denoiser_inputs()
            od, os_, _ = rbs[plane].denoise(sb.world_to_view(cam), sb.view_to_clip(cam), f, d["view_z"], d["normal_roughness"], d["diff"], d["spec"], motion=d["motion"],
                                            disocclusion_mix=d["disocclusion_mix"])
            td, ts = _device_image(od), _device_image(os_); torch.cuda.synchronize()
            b.denoiser_final_merge(plane, td.data_ptr(), ts.data_ptr()); b.synchronize()
        got, ref = a.readback_output_color().astype(np.float32), b.readback_output_color().astype(np.float32)
        assert np.isfinite(got).all()
        close = np.isclose(got, ref, rtol=1e-2, atol=2e-3).all(-1).mean()
        assert close > (0.985 if strict else 0.93), (strict, f, close)
        assert abs(got[..., :3].mean() - ref[..., :3].mean()) < 0.01 * ref[..., :3].mean(), (strict, f)
    for rb in rbs: rb.close()
    a.close(); b.close()


@pytest.mark.gpu
def test_tile_group_denoises_identically_after_the_setter(product):
    """realtime_mgpu.realtime_frame applies the settings on every rank: two contexts owning interleaved tiles give the frames one context gives with the same settings, bit for bit
    (without NEE-AT feedback every per-pixel step is deterministic)."""
    from rtxpt_b200 import scene_builder as sb, scenes, realtime_mgpu as M
    W, H = 160, 128
    scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    s = _settings(**CASES["all_changed"])
    k = sb.make_denoiser_constants(cam, hit_distance_parameters=tuple(s.hitDistanceParameters))
    def make(rank, world):
        c = product.Context(max_sub_samples_per_launch=1, tile_rank=rank, tile_world=world, tile_size=32); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
        c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2)); return c
    one = make(0, 1); two = [make(0, 2), make(1, 2)]; group = M.LocalGroup(two)
    one.set_reblur_settings(s)
    for f in range(3):
        consts.sampleBaseIndex = 2 * f
        for c in [one] + two: c.set_constants(consts)
        frame = sb.make_reblur_frame(cam, cam, frame_index=f)
        one.path_trace_realtime(False); one.denoise_realtime(k, frame); one.synchronize()
        M.realtime_frame(group, k, frame, reblur_settings=s)
        for c in two: c.synchronize()
        ref = dict(reblur=one.readback_reblur(), color=one.readback_output_color())
        for c in two:
            got = dict(reblur=c.readback_reblur(), color=c.readback_output_color())
            for name in ref["reblur"]: assert ref["reblur"][name].tobytes() == got["reblur"][name].tobytes(), (f, name)
            assert ref["color"].tobytes() == got["color"].tobytes(), f
    for c in [one] + two: c.close()
