"""GPU: NEE-AT temporal feedback of the CUDA path (neeat_kernels.cu, the NEEAT instantiations of the FILL shade and shadow kernels) against the oracle (oracle/pt_neeat.h).
The baker passes are reservoir / integer bookkeeping written with single IEEE operations: fed the same reservoirs they must reproduce the oracle bit for bit (their host build
already does, tests/test_neeat_port.py; here the atomics of P0, the device scan, the proxy fill and the cooperative tile sort join in).  The path-tracer side goes through libdevice
pow / the fast-math shading, so it is held to the estimator's properties: same mean as global-only sampling, lower error, and the oracle's own feedback statistics.

Tolerances marked "measured" come from GPU runs of these tests."""
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


def _pair(product, oracle, W, H, bays=7, strict=True, bounces=2):
    from rtxpt_b200 import scene_builder as sb, scenes
    scene, cam = scenes.light_gallery(W, H, bays=bays)
    consts = sb.make_constants(W, H, cam, bounce_count=bounces, diffuse_bounce_count=bounces); consts.NEEATFeedback = 1; consts.NEEATImportanceBoost = 3       # both importance boosters, as in RTXPT's UI
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam)); o.neeat_reset()
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=bounces, sub_samples=1); c.set_realtime(rt)
    return c, o, cam, consts, rt


def _same_state(c, o, W, H, n_lights, stage):
    P, B = W * H, ((W + 1) // 2) * ((H + 1) // 2)
    co, cp = o.neeat_raw(8, np.uint32, 8), c.neeat_raw(8, np.uint32, 8)
    assert np.array_equal(co, cp), (stage, co, cp)
    T = int(co[0]) * int(co[1]) * 128
    for what, n, name in ((0, P, "feedback weight"), (1, P, "feedback candidate"), (7, n_lights, "proxy counters"), (11, int(co[4]), "proxy table")) + \
                         (((2, P, "processed weight"), (3, P, "processed candidate"), (4, B, "blended weight"), (5, B, "blended candidate"), (6, T, "tile lists")) if stage == "end" else ()):
        a, b = o.neeat_raw(what, np.uint32, n), c.neeat_raw(what, np.uint32, n)
        assert len(a) == len(b) == n and np.array_equal(a, b), (stage, name, int((a != b).sum()))


@unverified
def test_baker_passes_reproduce_the_oracle(product, oracle):
    """Frame after frame both sides get the reservoirs the oracle's path tracer filled; everything the passes derive from them is identical."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 90, 58
    c, o, cam, consts, rt = _pair(product, oracle, W, H)
    n_lights = int(o.neeat_raw(12, np.uint32, 1)[0])
    for f in range(5):
        consts.sampleBaseIndex = f; c.set_constants(consts); o.set_constants(consts)
        if f > 0: c.neeat_set_feedback(o.neeat_raw(0, np.float32, W * H), o.neeat_raw(1, np.uint32, W * H))
        o.neeat_update_begin(); c.neeat_update_begin(); c.synchronize(); _same_state(c, o, W, H, n_lights, "begin")
        r = o.render_realtime(rt)                        # BUILD, update_end, FILL (inserts the feedback the next frame processes)
        c.path_trace_realtime(True); c.synchronize()     # same, on the GPU: its update_end saw the same inputs up to the depth guide
        g = c.readback_realtime()
        assert np.allclose(g["depth"], r["depth"], rtol=1e-5, atol=1e-6)
    # tile lists after the GPU's own update_end: well formed (sorted, run-length counts) even where a depth ulp flipped a reprojection decision
    lists = c.neeat_raw(6, np.uint32, 1 << 22).reshape(-1, 128); lights = lists >> 9; counts = (lists & 0x1FF) + 1
    assert (np.diff(lights.astype(np.int64), axis=1) >= 0).all() and lights.max() < n_lights
    for row_l, row_c in zip(lights[::5], counts[::5]):
        u, n = np.unique(row_l, return_counts=True)
        assert n.sum() == 128 and all((row_c[row_l == k] == m).all() for k, m in zip(u, n))
    c.close(); o.close()


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_feedback_loop_is_unbiased_and_helps(product, oracle, strict):
    """The whole loop on the GPU: the estimator's mean equals global-only sampling, the warmed-up error is lower, the feedback statistics match the oracle's."""
    from rtxpt_b200 import scene_builder as sb
    W, H = 112, 72
    c, o, cam, consts, rt = _pair(product, oracle, W, H, bays=10, strict=strict)
    fb = []
    for f in range(60):
        consts.sampleBaseIndex = f; c.set_constants(consts); c.neeat_update_begin(); c.path_trace_realtime(True); c.synchronize()
        fb.append(c.readback_output_color()[..., :3].astype(np.float32))
    valid_gpu = int(c.neeat_raw(8, np.uint32, 8)[7])
    fb = np.stack(fb)
    consts.NEEATFeedback = 0; gl = []
    for f in range(120):
        consts.sampleBaseIndex = f; c.set_constants(consts); c.path_trace_realtime(True); c.synchronize()
        gl.append(c.readback_output_color()[..., :3].astype(np.float32))
    gl = np.stack(gl); ref = gl.mean(0); warm = fb[12:]
    assert np.isfinite(fb).all()
    assert abs(warm.mean() / gl.mean() - 1) < 0.03
    assert np.abs(warm - ref).mean() < 0.95 * np.abs(gl - ref).mean()
    # the oracle's loop on the same scene reports a similar share of pixels with feedback
    consts.NEEATFeedback = 1
    for f in range(8):
        consts.sampleBaseIndex = f; o.set_constants(consts); o.neeat_update_begin(); o.render_realtime(rt)
    valid_cpu = int(o.neeat_raw(8, np.uint32, 8)[7])
    assert abs(valid_gpu - valid_cpu) < 0.1 * W * H, (valid_gpu, valid_cpu)
    c.close(); o.close()


@unverified
def test_neeat_api_errors(product):
    from rtxpt_b200 import scene_builder as sb, scenes
    W, H = 64, 48
    scene, cam = scenes.light_gallery(W, H, bays=4)
    consts = sb.make_constants(W, H, cam, bounce_count=2, diffuse_bounce_count=2); consts.NEEATFeedback = 1
    c = product.Context(max_sub_samples_per_launch=1); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=2, sub_samples=1))
    with pytest.raises(Exception): c.path_trace_realtime(True)               # update_begin missing
    with pytest.raises(Exception): c.path_trace(0, 1, False)                 # reference mode: update_begin / update_end missing (and this context exports no guides)
    c.neeat_update_begin(); c.path_trace_realtime(True); c.synchronize()
    with pytest.raises(Exception): c.neeat_update_end()                      # the frame's update_end already ran inside path_trace_realtime
    c.neeat_reset(); c.neeat_update_begin(); c.path_trace_realtime(True); c.synchronize()
    c.close()


@unverified
def test_reference_mode_feedback_loop(product, oracle):
    """Reference mode with feedback (RTXPT's default NEEType 2): update_begin, update_end on the guides the previous frame exported, one sub-sample per wavefront.  Unbiased
    against feedback-free sampling, lower error once warm, tile lists well formed."""
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    W, H = 112, 72
    scene, cam = scenes.light_gallery(W, H, bays=10)
    consts = sb.make_constants(W, H, cam, bounce_count=2, diffuse_bounce_count=2)
    c = product.Context(max_sub_samples_per_launch=4, flags=S.CFG_EXPORT_GUIDES); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    def frames(n, feedback):
        out = []
        consts.NEEATFeedback = 1 if feedback else 0
        for f in range(n):
            consts.sampleBaseIndex = 2 * f; c.set_constants(consts)
            if feedback: c.neeat_update_begin(); c.neeat_update_end()
            c.path_trace(0, 2, False); c.synchronize(); out.append(c.readback_output_color()[..., :3].astype(np.float32))
        return np.stack(out)
    consts.NEEATFeedback = 0; c.set_constants(consts); c.path_trace(0, 1, False); c.synchronize()        # a first frame leaves depth / motion guides behind
    fb = frames(48, True); gl = frames(96, False)
    ref = gl.mean(0); warm = fb[10:]
    assert np.isfinite(fb).all() and abs(warm.mean() / gl.mean() - 1) < 0.03
    assert np.abs(warm - ref).mean() < 0.95 * np.abs(gl - ref).mean()
    lists = c.neeat_raw(6, np.uint32, 1 << 22).reshape(-1, 128)
    assert (np.diff((lists >> 9).astype(np.int64), axis=1) >= 0).all()
    c.close()
