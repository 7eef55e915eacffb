"""GPU: rtxpt_b200_skin_register / rtxpt_b200_skin_update (skinning_kernels.cu) + the refit.  Tolerances marked "measured" come from GPU runs of these tests.  A context whose boxes were bent by a
two-joint skin must trace exactly like a fresh upload of the bent mesh (and like the oracle on it): the skin writes the same float positions a host-side blend produces.  Both libraries
link the IEEE build of the skinning kernels (csrc/Makefile), so every word of the shade records they rewrite must equal what the oracle's skin (oracle_skin) writes from the same inputs."""
import ctypes as C
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


@unverified
def test_skinned_boxes_trace_like_a_fresh_upload(product, oracle):
    from rtxpt_b200 import scenes, scene_builder as sb
    from test_gpu_refit import _rays
    from test_skinning import _run
    b = scenes.cornell_builder()
    scene = b.build()
    c = product.Context(); c.upload_scene(scene)
    # the third instance (the two boxes) has two geometries; skin the first: vertices above y = 0.8 follow joint 1, the rest joint 0
    g = b.meshes[b.instances[2][0]][0]
    pos = np.asarray(g["positions"], np.float32).reshape(-1, 3)
    ji = np.zeros((len(pos), 4), np.uint16); ji[pos[:, 1] > 0.8, 0] = 1
    jw = np.zeros((len(pos), 4), np.float32); jw[:, 0] = 1
    sid = c.skin_register(2, 0, pos, ji, jw)
    lean = np.eye(4, dtype=np.float32); lean[3, 0] = 0.35                       # joint 1: shift the top to +x
    mats = np.stack([np.eye(4, dtype=np.float32), lean])
    rays = _rays(20000, np.random.default_rng(4)); h0 = c.trace_rays(rays)
    c.skin_update(sid, mats); c.update_instance_transforms(np.stack([t for _, t in b.instances])); c.synchronize()
    got = c.trace_rays(rays)
    bent = pos.copy(); bent[pos[:, 1] > 0.8, 0] += np.float32(0.35)
    g["positions"] = bent; moved = b.build()
    o = oracle.Oracle(moved); want = o.trace_rays(rays); o.close()
    assert got.tobytes() == want.tobytes() and (got["t"] != h0["t"]).mean() > 0.005
    c.skin_update(sid, np.stack([np.eye(4, dtype=np.float32)] * 2)); c.update_instance_transforms(np.stack([t for _, t in b.instances])); c.synchronize()
    assert c.trace_rays(rays).tobytes() == h0.tobytes()
    c.close()


def _joints(rng, nv, joints, max_weights=4):
    """Joint indices and weights per vertex: 2 to `max_weights` non-zero weights (the rest 0, in random slots), summing to about 1."""
    ji = rng.integers(0, joints, (nv, 4)).astype(np.uint16)
    jw = rng.random((nv, 4)).astype(np.float32) + np.float32(0.05)
    k = rng.integers(2, max_weights + 1, nv)
    rank = np.argsort(rng.random((nv, 4)), 1)
    jw[rank >= k[:, None]] = 0                                                       # keeps k random slots of each vertex
    jw /= jw.sum(1, keepdims=True)
    return ji, jw


def _packed_frames(rng, nv):
    """Unit normals and tangents (both tangent signs) packed snorm8 x 4 as the vertex buffers hold them."""
    from test_skinning import _pack4
    n = rng.normal(0, 1, (nv, 3)); n /= np.linalg.norm(n, axis=1, keepdims=True); t = np.cross(n, rng.normal(0, 1, (nv, 3))); t /= np.linalg.norm(t, axis=1, keepdims=True)
    return _pack4(np.concatenate([n, np.zeros((nv, 1))], 1)), _pack4(np.concatenate([t, np.where(rng.random((nv, 1)) < 0.5, -1.0, 1.0)], 1))


def _oracle_records(oracle, records, first_gid, pos, nrm, tan, ji, jw, mats, idx):
    """oracle_skin on a copy of the read-back shade records (n x 24 words): the records it rewrites, and the skinned positions."""
    rec = records.copy(); op = np.zeros_like(pos); on = np.zeros(len(pos), np.uint32); ot = np.zeros(len(pos), np.uint32)
    f = oracle.lib().oracle_skin; f.argtypes = [C.c_uint32] * 3 + [C.c_void_p] * 11
    p = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data
    m = np.ascontiguousarray(mats, np.float32).reshape(-1, 16); idx = np.ascontiguousarray(idx, np.uint32)
    assert f(len(pos), len(idx), first_gid, p(pos), p(nrm), p(tan), p(ji), p(jw), p(m), p(idx), p(op), p(on), p(ot), p(rec)) == 0
    return rec, op


def _first_gid(records, sub_instance):
    """Global id of triangle 0 of a sub-instance (shade record word 22: sub-instance, word 23: triangle index within the geometry | flags)."""
    return int(np.nonzero((records[:, 22] == sub_instance) & ((records[:, 23] & 0x1FFFFFFF) == 0))[0][0])


def _corners(records, first, count):
    return records[first:first + count, [0, 1, 2, 4, 5, 6, 8, 9, 10]].view(np.float32)


def _sheet(nx, nz, size=1.2, origin=(1.5, 2.0, 1.5)):
    """A rippled nx x nz vertex grid (two triangles per cell)."""
    x, z = np.meshgrid(np.linspace(0, size, nx), np.linspace(0, size, nz), indexing="ij")
    pos = np.stack([x, 0.1 * np.sin(7 * x) * np.cos(5 * z), z], -1).reshape(-1, 3) + np.float64(origin)
    i = np.arange(nx * nz).reshape(nx, nz); a, b, c, d = i[:-1, :-1].ravel(), i[1:, :-1].ravel(), i[1:, 1:].ravel(), i[:-1, 1:].ravel()
    return pos.astype(np.float32), np.concatenate([np.stack([a, b, c], 1), np.stack([a, c, d], 1)]).astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_skin_records_equal_the_oracle_word_for_word(product, oracle, strict):
    from rtxpt_b200 import scenes, scene_builder as sb
    from test_skinning import _mats
    rng = np.random.default_rng(31)
    pos, idx = _sheet(450, 451)                                                                  # 202 950 vertices, 404 100 triangles: neither a multiple of 256
    nv, nt = len(pos), len(idx)
    assert nv >= 200_000 and nv % 256 and nt % 256
    nrm, tan = _packed_frames(rng, nv)
    ji, jw = _joints(rng, nv, 64)
    assert (jw == 0).any() and ((jw > 0).sum(1) == 4).any()
    b = scenes.cornell_builder(); white = 0
    b.add_instance(b.add_mesh([dict(positions=pos, indices=idx, normals=np.tile(np.float32([0, 1, 0]), (nv, 1)), uvs=np.zeros((nv, 2), np.float32),
                                      tangents=np.tile(np.float32([1, 0, 0, 1]), (nv, 1)), material=white)]), sb.identity34())
    scene = b.build()
    c = product.Context(strict=strict); c.upload_scene(scene)
    rec0 = c.scene_raw(2); sub = scene.instances[3].firstGeometryInstanceIndex; first = _first_gid(rec0, sub)
    assert len(c.scene_raw(3)) == 0
    sid = c.skin_register(3, 0, pos, ji, jw, nrm, tan)
    assert np.array_equal(c.scene_raw(2), rec0)
    prev = c.scene_raw(3); assert np.array_equal(prev.view(np.uint32), _corners(rec0, first, nt).view(np.uint32))          # registered: no motion yet
    want = rec0
    for step in range(2):
        mats = _mats(rng, 64)
        before = want
        want, op = _oracle_records(oracle, before, first, pos, nrm, tan, ji, jw, mats, idx)
        c.skin_update(sid, mats)
        got = c.scene_raw(2)
        bad = np.nonzero((got != want).any(1))[0]
        assert len(bad) == 0, (step, len(bad), bad[:4], got[bad[:1]], want[bad[:1]])
        assert np.array_equal(got[:first], rec0[:first]) and np.array_equal(got[first + nt:], rec0[first + nt:])        # every other geometry untouched
        assert np.array_equal(c.scene_raw(3).view(np.uint32), _corners(before, first, nt).view(np.uint32))               # the corners from before this update
        assert not np.array_equal(got[first:first + nt, 18:21], rec0[first:first + nt, 18:21]) and np.array_equal(got[first:first + nt, 12:18], rec0[first:first + nt, 12:18])
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_skin_of_an_offset_geometry_in_a_second_instance(product, oracle, strict):
    """The tall box (geometry 1 of the boxes mesh: non-zero index and position offsets) of a second instance of that mesh; the first instance's records stay as uploaded."""
    from rtxpt_b200 import scenes, scene_builder as sb
    from test_skinning import _mats
    rng = np.random.default_rng(32)
    b = scenes.cornell_builder(); boxes = b.instances[2][0]
    b.add_instance(boxes, sb.translate_scale((0.3, 0.0, -0.4)))
    scene = b.build()
    g = scene.geometries[scene.instances[3].firstGeometryIndex + 1]
    assert g.indexOffset > 0 and g.positionOffset > 0
    geo = b.meshes[boxes][1]; pos = np.asarray(geo["positions"], np.float32).reshape(-1, 3); idx = np.asarray(geo["indices"], np.uint32).reshape(-1, 3)
    nrm, tan = _packed_frames(rng, len(pos)); ji, jw = _joints(rng, len(pos), 4)
    c = product.Context(strict=strict); c.upload_scene(scene)
    rec0 = c.scene_raw(2); first = _first_gid(rec0, scene.instances[3].firstGeometryInstanceIndex + 1)
    sid = c.skin_register(3, 1, pos, ji, jw, nrm, tan)
    mats = _mats(rng, 4)
    want, _ = _oracle_records(oracle, rec0, first, pos, nrm, tan, ji, jw, mats, idx)
    c.skin_update(sid, mats)
    got = c.scene_raw(2)
    assert np.array_equal(got, want) and not np.array_equal(got, rec0)
    assert np.array_equal(c.scene_raw(3).view(np.uint32), _corners(rec0, first, len(idx)).view(np.uint32))
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_second_skin_keeps_the_earlier_previous_position_ranges(product, oracle, strict):
    """A scene uploaded with a previous-position stream (the short box), then two skins registered one after the other: each registration regrows the previous-position
    buffer, and the ranges already in it must survive; an update writes only its own skin's range."""
    from test_motion_vectors import _builder
    from test_skinning import _mats
    rng = np.random.default_rng(33)
    b0 = _builder(); short = np.asarray(b0.meshes[b0.instances[2][0]][0]["positions"], np.float32).reshape(-1, 3)
    b = _builder(short_prev_positions=short + np.float32([0.05, 0, 0])); scene = b.build()
    c = product.Context(strict=strict); c.upload_scene(scene)
    rec0 = c.scene_raw(2); stream = c.scene_raw(3)
    assert len(stream) == np.asarray(b.meshes[b.instances[2][0]][0]["indices"]).size // 3
    skins = []
    for inst, geom in ((2, 1), (0, 1)):                                                          # the tall box, then the room's left wall
        geo = b.meshes[b.instances[inst][0]][geom]; pos = np.asarray(geo["positions"], np.float32).reshape(-1, 3); idx = np.asarray(geo["indices"], np.uint32).reshape(-1, 3)
        ji, jw = _joints(rng, len(pos), 3)
        before = c.scene_raw(3)
        sid = c.skin_register(inst, geom, pos, ji, jw)
        after = c.scene_raw(3)
        first = _first_gid(rec0, scene.instances[inst].firstGeometryInstanceIndex + geom)
        assert len(after) == len(before) + len(idx) and np.array_equal(after[:len(before)].view(np.uint32), before.view(np.uint32))
        assert np.array_equal(after[len(before):].view(np.uint32), _corners(rec0, first, len(idx)).view(np.uint32))
        skins.append((sid, first, len(before), pos, ji, jw, idx))
    assert np.array_equal(c.scene_raw(3)[:len(stream)], stream)
    records = rec0
    for sid, first, base, pos, ji, jw, idx in skins:
        mats = _mats(rng, 3); prev_all = c.scene_raw(3)
        want, _ = _oracle_records(oracle, records, first, pos, None, None, ji, jw, mats, idx)
        c.skin_update(sid, mats)
        got = c.scene_raw(2); assert np.array_equal(got, want); records = got
        now = c.scene_raw(3); mine = slice(base, base + len(idx))
        assert np.array_equal(now[mine].view(np.uint32), prev_all[mine].view(np.uint32))          # no motion since registration: the corners as they were
        rest = np.ones(len(now), bool); rest[mine] = False
        assert np.array_equal(now[rest], prev_all[rest])
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_blended_skin_and_rigid_move_trace_like_the_oracle(product, oracle, strict):
    """A blended skin of the short box and a new matrix of its instance, then the refit: hits equal the oracle's on a scene built from oracle_skin's positions under that matrix."""
    from rtxpt_b200 import scenes
    from test_gpu_parity import hits_bit_equal, random_rays
    from test_gpu_refit import about, rotation, instance_centres
    from test_skinning import _mats
    rng = np.random.default_rng(34)
    b = scenes.cornell_builder(); scene = b.build()
    geo = b.meshes[b.instances[2][0]][0]; pos = np.asarray(geo["positions"], np.float32).reshape(-1, 3); idx = np.asarray(geo["indices"], np.uint32).reshape(-1, 3)
    ji, jw = _joints(rng, len(pos), 4)
    mats = _mats(rng, 4); mats[:, 3, :3] *= np.float32(0.1)                                      # rotating joints, short offsets
    boxes = about(rotation((1, 2, -1), 0.35) @ np.diag([1.0, 1.0, -1.0]), instance_centres(scene)[2], (0.1, 0.0, 0.2))
    c = product.Context(strict=strict); c.upload_scene(scene)
    rec0 = c.scene_raw(2)
    sid = c.skin_register(2, 0, pos, ji, jw)
    c.skin_update(sid, mats); c.update_instance_transforms(np.stack([b.instances[0][1], b.instances[1][1], boxes]))
    _, skinned = _oracle_records(oracle, rec0, 0, pos, None, None, ji, jw, mats, idx)
    geo["positions"] = skinned; b.instances[2] = (b.instances[2][0], boxes); moved = b.build()
    rays = random_rays(rng, 300000, [0.1, 0.1, -4.0], [5.4, 5.4, 5.4])
    o = oracle.Oracle(moved)
    a, w = c.trace_rays(rays), o.trace_rays(rays)
    assert hits_bit_equal(a, w).all() and ((w["inst"] == 2) & (w["geom"] == 0) & (w["t"] >= 0)).mean() > 0.005
    rays[:, 7] = rng.uniform(0.5, 40.0, len(rays)).astype(np.float32)
    assert np.array_equal(c.trace_rays(rays, any_hit=True)["t"] >= 0, o.trace_rays(rays, any_hit=True)["t"] >= 0)
    o.close(); c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_motion_vectors_of_a_blended_skin(product, oracle, strict):
    """Step 3 of test_motion_vectors.test_gpu_motion_vectors_after_instance_update_and_skinning with rotating joints and two to four weights per vertex.  Registered without normals,
    so the oracle's scene (bent positions, bind-pose normals, previous positions = the bind pose) is the surface the context holds."""
    from rtxpt_b200 import scene_builder as sb
    from test_motion_vectors import W, H, _builder, _pair, _compare_motion
    from test_skinning import _mats
    rng = np.random.default_rng(35)
    b = _builder(); scene = b.build()
    cam = sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    consts = sb.make_constants(W, H, cam, bounce_count=8, diffuse_bounce_count=3); rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam)); c.set_realtime(rt)
    geo = b.meshes[b.instances[2][0]][0]; pos = np.asarray(geo["positions"], np.float32).reshape(-1, 3); idx = np.asarray(geo["indices"], np.uint32).reshape(-1, 3)
    ji, jw = _joints(rng, len(pos), 4)
    mats = _mats(rng, 4); mats[:, 3, :3] *= np.float32(0.1)
    ident = sb.identity34(); xf = np.stack([ident, ident, ident])
    rec0 = c.scene_raw(2)
    sid = c.skin_register(2, 0, pos, ji, jw)
    c.skin_update(sid, mats); c.update_instance_transforms(xf); c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
    _, bent = _oracle_records(oracle, rec0, _first_gid(rec0, scene.instances[2].firstGeometryInstanceIndex), pos, None, None, ji, jw, mats, idx)
    bs = _builder(short_prev_positions=pos); bs.meshes[bs.instances[2][0]][0]["positions"] = bent
    _, _, _, o, _ = _pair(oracle, bs); r = o.render_realtime(rt); o.close()
    mv = _compare_motion(g, r, strict); assert (np.abs(mv[..., :2]).max(-1) > 0.05).mean() > 0.01
    c.close()
