"""Motion vectors of moving and skinned geometry in the BUILD pass, and the curvature heuristics of PSDBlockMotionVectorsAtSurfaceType 1 / 2 (SURVEY §8 row a17):
Bridge::loadSurface's prevPosW = instance.prevTransform x last frame's object-space position (PathTracerBridgeDonut.hlsli:187-199, :631), the world motion carried through the stacked
reflections (PathTracerStablePlanes.hlsli:282-291) and the block decision (BridgeDonut:702-718, Libraries/MicroRng.hlsli).  CPU: the oracle against the analytic screen-space motion;
GPU: the CUDA path against the oracle, after rtxpt_b200_update_instance_transforms / rtxpt_b200_skin_update and for a scene uploaded with a previous-position stream."""
import numpy as np
import pytest

W, H = 96, 96


def _builder(boxes_prev=None, short_prev_positions=None, block_type=0, curved=False):
    """Cornell box; boxes_prev: last frame's matrix of the boxes instance; short_prev_positions: previous-position stream of the short box; block_type / curved: a
    sphere with the given PSDBlockMotionVectorsAtSurfaceType in place of nothing (for the heuristics)."""
    from rtxpt_b200 import scenes, scene_builder as sb
    b = scenes.cornell_builder(delta_surfaces=False)         # diffuse boxes: the surface a pixel exports is the box itself (behind a mirror or glass it would be what they show)
    if boxes_prev is not None: b.prev_transforms = {2: np.float32(boxes_prev).reshape(3, 4)}
    if short_prev_positions is not None: b.meshes[b.instances[2][0]][0]["prev_positions"] = short_prev_positions
    if curved:
        m = b.add_material(sb.Material(base_color=(0.9, 0.9, 0.9), roughness=0.0, metalness=1.0, psd_exclude=False, psd_dominant_delta_lobe=1, psd_block_mvs_at_surface=block_type))
        b.add_instance(b.add_mesh([scenes._uv_sphere((1.4, 3.6, 1.8), 0.7, 24, 16, m)]), sb.identity34())
    return b


def _pair(oracle, b):
    from rtxpt_b200 import scene_builder as sb
    scene = b.build(); cam = sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3)
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1)
    return scene, cam, consts, o, rt


def _project(cam, p):
    from rtxpt_b200 import scene_builder as sb
    m = np.asarray(sb.world_to_clip(cam), np.float64).reshape(4, 4)
    c = np.concatenate([p, np.ones(p.shape[:-1] + (1,))], -1) @ m
    return np.stack([(c[..., 0] / c[..., 3] * 0.5 + 0.5) * W, (0.5 - c[..., 1] / c[..., 3] * 0.5) * H], -1), c[..., 3]


def test_oracle_motion_of_a_moved_instance_is_the_projected_displacement(oracle):
    from rtxpt_b200 import scene_builder as sb
    shift = np.float32([0.30, 0.0, -0.20])
    prev = sb.identity34().copy(); prev[:, 3] = -shift                        # last frame the boxes stood `shift` further back: they moved by +shift since
    scene, cam, consts, o, rt = _pair(oracle, _builder(boxes_prev=prev))
    r = o.render_realtime(rt); o.close()
    _, _, _, o0, _ = _pair(oracle, _builder()); r0 = o0.render_realtime(rt); o0.close()
    mv, mv0 = r["motion"].astype(np.float32), r0["motion"].astype(np.float32)
    assert np.abs(mv0[..., :2]).max() < 1e-3                                  # static scene, static camera: no motion anywhere
    moving = np.abs(mv[..., :2]).max(-1) > 1e-2
    assert 0.05 < moving.mean() < 0.6                                         # the boxes (and what the mirror / glass show of themselves), not the room
    # first-hit pixels on the boxes: world position from depth along the camera ray; its previous position is `shift` back; motion = difference of the projections
    ys, xs = np.nonzero(moving & (r["header"][3] & 3 == 0) & (r["depth"] > 0))
    # the guide's depth is the camera-space distance along the ray; reconstruct through the inverse view-projection instead of trusting conventions: use the identity
    # motion == project(p - shift) - project(p) for SOME p on the pixel's ray; solve for the ray parameter by matching the guide's own z component (w' - w)
    cam_pos = np.float64(cam.PosW[:]); m = np.asarray(sb.world_to_clip(cam), np.float64).reshape(4, 4)
    checked = 0
    for y, x in list(zip(ys, xs))[::7]:
        ndc = np.float64([(x + 0.5) / W * 2 - 1, 1 - (y + 0.5) / H * 2, 0.5, 1.0]); far = ndc @ np.linalg.inv(m); far = far[:3] / far[3]
        d = far - cam_pos; d /= np.linalg.norm(d)
        best = None
        for t in np.linspace(5.0, 16.0, 221):
            p = cam_pos + d * t; (s1, w1), (s0, w0) = _project(cam, p - np.float64(shift)), _project(cam, p)
            err = np.abs((s1 - s0) - mv[y, x, :2]).max()
            if best is None or err < best[0]: best = (err, w1 - w0)
        assert best[0] < 0.06, (x, y, best, mv[y, x])                         # fp16 guide, coarse t search
        assert abs(best[1] - mv[y, x, 2]) < 0.02
        checked += 1
    assert checked > 20


def test_oracle_previous_position_stream_and_block_heuristics(oracle):
    from rtxpt_b200 import scenes
    b = _builder()
    pos = np.asarray(b.meshes[b.instances[2][0]][0]["positions"], np.float32).reshape(-1, 3)
    prev = pos.copy(); prev[pos[:, 1] > 0.8, 0] -= np.float32(0.35)          # last frame the top of the short box leaned 0.35 to -x
    scene, cam, consts, o, rt = _pair(oracle, _builder(short_prev_positions=prev)); r = o.render_realtime(rt); o.close()
    mv = r["motion"].astype(np.float32)
    moving = np.abs(mv[..., 0]) > 0.05
    top = np.float64([1.8, 1.65, 1.7]); (s_prev, _), (s_now, _) = _project(cam, top - np.float64([0.35, 0, 0])), _project(cam, top)
    want = np.sign(s_prev[0] - s_now[0])                                      # which way a point of the box's top came from on screen
    assert 0.01 < moving.mean() < 0.3 and (np.sign(mv[..., 0][moving]) == want).mean() > 0.95
    assert abs(np.abs(mv[..., 0]).max() - abs(s_prev[0] - s_now[0])) < 0.25 * abs(s_prev[0] - s_now[0])       # the top edge moves by about the analytic amount (perspective varies over the box)
    # block types on a curved mirror: Off lets the mirror's reflections define the surface seen (motion vectors / depth of what is reflected), Full stops at the sphere; the
    # automatic modes stop where the triangle's normal gradient x ray-cone width exceeds a threshold jittered by MicroRng: AutoHigh (0.0005) blocks at least where AutoLow (0.03) does
    depth = {}
    for bt in (0, 1, 2, 3):
        scene, cam, consts, o, rt = _pair(oracle, _builder(block_type=bt, curved=True)); depth[bt] = o.render_realtime(rt)["depth"].copy(); o.close()
    sphere = depth[3] != depth[0]                                             # pixels whose exported surface changes when the sphere blocks
    assert 0.01 < sphere.mean() < 0.2
    blocked1, blocked2 = (depth[1] == depth[3]) & sphere, (depth[2] == depth[3]) & sphere
    assert blocked2.sum() >= blocked1.sum() and blocked2.sum() > 0.9 * sphere.sum()
    assert ((depth[1] == depth[0]) | (depth[1] == depth[3]))[sphere].all()    # every pixel takes one of the two outcomes


def _compare_motion(g, r, strict):
    same = (g["header"][:3] == r["header"][:3]).all(0)
    assert same.mean() > 0.995
    a, b = g["motion"].astype(np.float32)[same], r["motion"].astype(np.float32)[same]
    if strict: assert (a == b).all(-1).mean() > 0.995, (a == b).all(-1).mean()
    assert np.isclose(a, b, rtol=2e-3, atol=2e-3).all(-1).mean() > 0.995
    assert np.allclose(g["depth"][same], r["depth"][same], rtol=1e-5, atol=1e-6)
    return b


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [True, False])
def test_gpu_motion_vectors_after_instance_update_and_skinning(product, oracle, strict):
    from rtxpt_b200 import scene_builder as sb
    ident = sb.identity34(); moved = ident.copy(); moved[:, 3] = (0.30, 0.0, -0.20)
    b = _builder(); scene = b.build()
    cam = sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3); rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam)); c.set_realtime(rt)
    # 1. rigid motion: the boxes move by +0.3 x, -0.2 z; the instance table keeps last frame's matrix
    c.update_instance_transforms(np.stack([ident, ident, moved])); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    bm = _builder(boxes_prev=ident); bm.instances[2] = (bm.instances[2][0], moved)
    _, _, _, o, _ = _pair(oracle, bm); r = o.render_realtime(rt); o.close()
    mv = _compare_motion(g, r, strict); assert (np.abs(mv[..., :2]).max(-1) > 1e-2).mean() > 0.05
    # 2. the same matrices again: nothing moved since last frame
    c.update_instance_transforms(np.stack([ident, ident, moved])); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    assert np.abs(g["motion"].astype(np.float32)[..., :2]).max() < 1e-3
    # 2b. a rotation about an oblique axis and a mirror (det < 0) about the boxes' centre: normals go through xfVector of a matrix that flips the winding
    from test_gpu_refit import about, rotation
    turned = about(rotation((1.0, 2.0, -0.7), 0.35) @ np.diag([-1.0, 1.0, 1.0]), (2.77, 1.2, 2.6), (0.1, 0.0, 0.1))
    c.update_instance_transforms(np.stack([ident, ident, turned])); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    bm = _builder(boxes_prev=moved); bm.instances[2] = (bm.instances[2][0], turned)
    _, _, _, o, _ = _pair(oracle, bm); r = o.render_realtime(rt); o.close()
    mv = _compare_motion(g, r, strict); assert (np.abs(mv[..., :2]).max(-1) > 1e-2).mean() > 0.05
    # 3. skinning: the top of the short box leans 0.35 to +x; the records' old corners become the previous-position stream
    c.update_instance_transforms(np.stack([ident, ident, ident]))
    geo = b.meshes[b.instances[2][0]][0]; pos = np.asarray(geo["positions"], np.float32).reshape(-1, 3)
    ji = np.zeros((len(pos), 4), np.uint16); ji[pos[:, 1] > 0.8, 0] = 1; jw = np.zeros((len(pos), 4), np.float32); jw[:, 0] = 1
    sid = c.skin_register(2, 0, pos, ji, jw)
    lean = np.eye(4, dtype=np.float32); lean[3, 0] = 0.35
    c.update_instance_transforms(np.stack([ident, ident, ident])); c.path_trace_realtime(True); c.synchronize()
    assert np.abs(c.readback_realtime()["motion"].astype(np.float32)[..., :2]).max() < 1e-3          # registered, not yet moved
    c.skin_update(sid, np.stack([np.eye(4, dtype=np.float32), lean])); c.update_instance_transforms(np.stack([ident, ident, ident])); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    bent = pos.copy(); bent[pos[:, 1] > 0.8, 0] += np.float32(0.35)
    bs = _builder(short_prev_positions=pos); bs.meshes[bs.instances[2][0]][0]["positions"] = bent
    _, _, _, o, _ = _pair(oracle, bs); r = o.render_realtime(rt); o.close()
    mv = _compare_motion(g, r, strict); assert (np.abs(mv[..., 0]) > 0.05).mean() > 0.01
    c.close()


@pytest.mark.gpu
def test_gpu_previous_position_stream_at_upload_and_block_heuristics(product, oracle):
    from rtxpt_b200 import scene_builder as sb
    b0 = _builder(); pos = np.asarray(b0.meshes[b0.instances[2][0]][0]["positions"], np.float32).reshape(-1, 3)
    prev = pos.copy(); prev[pos[:, 1] > 0.8, 0] -= np.float32(0.35)
    for kw in (dict(short_prev_positions=prev), dict(block_type=1, curved=True), dict(block_type=2, curved=True)):
        scene, cam, consts, o, rt = _pair(oracle, _builder(**kw)); r = o.render_realtime(rt); o.close()
        c = product.Context(max_sub_samples_per_launch=1, strict=True); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam)); c.set_realtime(rt)
        c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime(); c.close()
        _compare_motion(g, r, True)
