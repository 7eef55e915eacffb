"""GPU: rtxpt_b200_update_instance_transforms (refit_kernels.cu).  Tolerances marked "measured" come from GPU runs of these tests.  The refit re-transforms the leaf triangles with the arithmetic of the
scene upload, so a refitted context must trace exactly like a context (and an oracle) that was given the moved scene from the start.  Both libraries link the IEEE build of the refit
kernels (csrc/Makefile), so every word they write must equal what the host build of the same bodies (tests/emu: emu_refit) writes from the same inputs."""
import copy
import ctypes as C
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


def _cornell_with(transforms):
    """The Cornell box with its three instances (room, lamp, boxes) placed by `transforms`."""
    from rtxpt_b200 import scenes, scene_builder as sb
    b = scenes.cornell_builder()
    b.instances = [(mesh, np.float32(t).reshape(3, 4)) for (mesh, _), t in zip(b.instances, transforms)]
    return b.build()


def _rays(n, rng):
    o = np.tile(np.float32([2.78, 2.73, -8.0]), (n, 1)); d = rng.normal(0, 1, (n, 3)).astype(np.float32); d[:, 2] = np.abs(d[:, 2]) + 1.5; d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = np.zeros((n, 8), np.float32); r[:, 0:3] = o; r[:, 3] = 0.0; r[:, 4:7] = d; r[:, 7] = 1e30
    return r


def rotation(axis, angle):
    ax = np.float64(axis) / np.linalg.norm(axis); K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def about(A, pivot, t=(0, 0, 0)):
    """3x4 float32 matrix applying the 3x3 `A` about `pivot`, then translating by `t`."""
    p = np.float64(pivot)
    return np.float32(np.hstack([A, (p - A @ p + np.float64(t))[:, None]]))


def instance_centres(scene):
    """World-space centre of each instance's bounding box (from the scene's vertex buffers and matrices)."""
    out = []
    for ii in range(scene.desc.instanceCount):
        inst = scene.instances[ii]; lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
        for k in range(inst.numGeometries):
            g = scene.geometries[inst.firstGeometryIndex + k]
            v = np.ctypeslib.as_array((C.c_float * (g.numVertices * 3)).from_address(scene.buffers[g.vertexBufferIndex].data + g.positionOffset)).reshape(-1, 3)
            lo, hi = np.minimum(lo, v.min(0)), np.maximum(hi, v.max(0))
        m = np.float64(inst.transform[:]).reshape(3, 4); out.append(m[:, :3] @ ((lo + hi) / 2) + m[:, 3])
    return np.array(out)


def mixed_motion(scene, fixed=(), far=False, start=0):
    """One matrix per instance, cycling (from `start`) through identity, a rotation about an oblique axis, a non-uniform scale, a mirror (det < 0) and a translation (of 10^4 with
    far=True, else a short one), each about the instance's own centre; instances listed in `fixed` keep their uploaded matrix."""
    out = []
    for ii, c in enumerate(instance_centres(scene)):
        R = rotation((1.0, 2.0 + ii, -0.5), 0.3 + 0.1 * ii); k = (ii + start) % 5
        if ii in fixed or k == 0: A, t = np.eye(3), (0, 0, 0)
        elif k == 1: A, t = R, (0.2, 0.1, -0.3)
        elif k == 2: A, t = R @ np.diag([1.3, 0.6, 1.1]), (0, 0.15, 0)
        elif k == 3: A, t = R @ np.diag([-1.0, 1.0, 1.0]), (-0.1, 0, 0.2)
        else: A, t = rotation((0.3, 1.0, 0.2), 0.2), ((1e4, 0, 0) if far else (0.3, 0, 0.3))
        base = np.float64(scene.instances[ii].transform[:]).reshape(3, 4)
        m = np.float64(about(A, c, t)); out.append(np.float32(np.hstack([m[:, :3] @ base[:, :3], (m[:, :3] @ base[:, 3] + m[:, 3])[:, None]])))
    return np.stack(out)


def moved_scene(scene, transforms):
    """A shallow copy of `scene` whose instance table carries `transforms` (the geometry, materials and textures are shared)."""
    from rtxpt_b200 import structs as S
    s = copy.copy(scene); n = scene.desc.instanceCount
    s.instances = (S.InstanceData * max(1, n))(); C.memmove(s.instances, scene.instances, C.sizeof(S.InstanceData) * n)
    for i in range(n): s.instances[i].transform[:] = np.float32(transforms[i]).reshape(12).tolist()
    s.desc = S.SceneDesc.from_buffer_copy(scene.desc); s.desc.instances = s.instances
    return s


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def strided_city():
    """The city at 3.68 M triangles: both refit kernels need more than one grid pass on an H100 (asserted from the uploaded tree by the test)."""
    from rtxpt_b200 import scenes
    return scenes.city_block(target_triangles=3_600_000, texture_size=64, n_textures=4)[0]


@unverified
def test_refit_traces_like_a_fresh_upload(product, oracle):
    from rtxpt_b200 import scene_builder as sb
    rng = np.random.default_rng(3)
    ident = sb.identity34()
    a = 0.5; moved_boxes = np.float32([[np.cos(a), 0, np.sin(a), 0.6], [0, 1, 0, 0.0], [-np.sin(a), 0, np.cos(a), 0.9]])
    base = _cornell_with([ident, ident, ident]); moved = _cornell_with([ident, ident, moved_boxes])
    c = product.Context(); c.upload_scene(base)
    rays = _rays(20000, rng)
    h0 = c.trace_rays(rays)
    c.update_instance_transforms(np.stack([ident, ident, ident])); c.synchronize()
    assert c.trace_rays(rays).tobytes() == h0.tobytes()                                         # identity refit: the built tree, bit for bit
    c.update_instance_transforms(np.stack([ident, ident, moved_boxes])); c.synchronize()
    got = c.trace_rays(rays); got_any = c.trace_rays(rays, any_hit=True)
    o = oracle.Oracle(moved); want = o.trace_rays(rays); o.close()
    assert got.tobytes() == want.tobytes()                                                       # hit records: bit-exact class, like the parity tests of the static path
    assert np.array_equal(got_any["t"] >= 0, want["t"] >= 0)
    assert (got["t"] != h0["t"]).mean() > 0.02                                                   # the boxes did move
    c2 = product.Context(); c2.upload_scene(moved); assert c2.trace_rays(rays).tobytes() == got.tobytes(); c2.close()
    c.update_instance_transforms(np.stack([ident, ident, ident])); c.synchronize()
    assert c.trace_rays(rays).tobytes() == h0.tobytes()                                          # and back
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_refit_equals_the_host_build_where_the_launch_strides(product, strided_city, strict):
    import host_build_lib as emu
    from test_refit import _refit
    scene = strided_city
    c = product.Context(strict=strict); c.upload_scene(scene)
    nodes0, tris0, rec0, levels = c.scene_raw(0), c.scene_raw(1), c.scene_raw(2), c.scene_raw(5)
    assert len(c.scene_raw(6)) == 0 and levels[-1] == len(nodes0) and len(rec0) == len(tris0)
    # refit_kernels.cu: k_refit_tris runs smCount x 8 x 256 threads, k_refit_level at most smCount x 16 x 128 per level; this tree must need a second grid pass of both
    sm = sm_count(); tri_grid, level_grid = sm * 8 * 256, sm * 16 * 128
    largest = int(np.diff(levels.astype(np.int64)).max())
    print(f"\n{len(tris0)} triangles, {len(nodes0)} nodes in {len(levels) - 1} levels, largest level {largest} nodes; {sm} SMs: k_refit_tris grid {tri_grid} threads, k_refit_level grid {level_grid} threads")
    assert len(tris0) > tri_grid and largest > level_grid
    ident = np.stack([np.float32(scene.instances[i].transform[:]).reshape(3, 4) for i in range(scene.desc.instanceCount)])
    mats = mixed_motion(scene, far=True)
    assert sum(np.linalg.det(np.float64(m[:, :3])) < 0 for m in mats) >= 1 and sum(np.array_equal(m, i) for m, i in zip(mats, ident)) >= 1 and np.abs(mats[:, :, 3]).max() > 5e3
    # an identity refit right after upload returns the built tree, and its exact boxes are the host build's
    c.update_instance_transforms(ident)
    n1, t1, b1 = c.scene_raw(0), c.scene_raw(1), c.scene_raw(6)
    assert np.array_equal(n1, nodes0) and np.array_equal(t1, tris0)
    _, _, want_b1 = _refit(emu, nodes0, tris0, rec0, ident, levels)
    assert np.array_equal(b1.view(np.uint32), want_b1.view(np.uint32))
    # every instance on its own matrix: nodes, leaf triangles and exact boxes equal the host build word for word; the shade records are not the refit's business
    want_n, want_t, want_b = _refit(emu, nodes0, tris0, rec0, mats, levels)
    assert not np.array_equal(want_n, nodes0)
    for _ in range(2):                                                                              # the same matrices twice: the same words
        c.update_instance_transforms(mats)
        n2, t2, b2 = c.scene_raw(0), c.scene_raw(1), c.scene_raw(6)
        assert np.array_equal(t2, want_t) and np.array_equal(n2, want_n) and np.array_equal(b2.view(np.uint32), want_b.view(np.uint32))
        assert np.array_equal(c.scene_raw(2), rec0)
    inst = c.scene_raw(4)
    assert all(np.array_equal(np.float32(inst[i].transform[:]), mats[i].reshape(12)) and np.array_equal(np.float32(inst[i].prevTransform[:]), mats[i].reshape(12)) for i in range(len(mats)))
    # and back: the uploaded tree, bit for bit
    c.update_instance_transforms(ident)
    assert np.array_equal(c.scene_raw(0), nodes0) and np.array_equal(c.scene_raw(1), tris0)
    c.close()


def _targets(scene, transforms, rng, n):
    """`n` world-space vertices of the moved scene: vertices of every instance's first geometry under its new matrix."""
    pts = []
    for ii in range(scene.desc.instanceCount):
        inst = scene.instances[ii]; g = scene.geometries[inst.firstGeometryIndex]
        v = np.ctypeslib.as_array((C.c_float * (g.numVertices * 3)).from_address(scene.buffers[g.vertexBufferIndex].data + g.positionOffset)).reshape(-1, 3).astype(np.float64)
        m = np.float64(transforms[ii]); pts.append(v[rng.integers(0, len(v), n // scene.desc.instanceCount + 1)] @ m[:, :3].T + m[:, 3])
    return np.concatenate(pts)[:n]


def _rays_at(origin, targets):
    """Unnormalised directions from `origin` through each target (rays that graze shared vertices and edges)."""
    org = np.tile(np.float32(origin), (len(targets), 1))
    return np.concatenate([org, np.zeros((len(targets), 1), np.float32), (targets - org).astype(np.float32), np.full((len(targets), 1), 1e15, np.float32)], 1).astype(np.float32)


def _box_and_origin(which):
    return (([0.1, 0.1, -4.0], [5.4, 5.4, 5.4]), [2.7, 2.7, -3.0]) if which == "cornell" else (([-110, 0.1, -110], [110, 45, 110]), [3.0, 60.0, -5.0])


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("which", ["cornell", "city"])
def test_refitted_tree_traces_like_the_oracle(product, oracle, cornell, small_city, monkeypatch, strict, which):
    from test_gpu_parity import hits_bit_equal, random_rays
    scene = (cornell if which == "cornell" else small_city)[0]
    mats = mixed_motion(scene, start=2 if which == "cornell" else 0)          # Cornell: the room scaled, the lamp mirrored, the boxes rotated and moved
    moved = moved_scene(scene, mats)
    o = oracle.Oracle(moved); fresh = product.Context(strict=strict); fresh.upload_scene(moved)
    (lo, hi), origin = _box_and_origin(which)
    for smem in (None, "200"):                                                                      # 200: the top of the tree is staged in shared memory (read at context creation)
        if smem: monkeypatch.setenv("RTXPT_SMEM_NODES", smem)
        rng = np.random.default_rng(21)
        c = product.Context(strict=strict); c.upload_scene(scene)
        rays = random_rays(rng, 300000, lo, hi)
        before = c.trace_rays(rays)
        c.update_instance_transforms(mats)
        a, b = c.trace_rays(rays), o.trace_rays(rays)
        assert hits_bit_equal(a, b).all() and hits_bit_equal(a, fresh.trace_rays(rays)).all()
        assert (a["t"] != before["t"]).mean() > 0.05
        edge = _rays_at(origin, _targets(scene, mats, rng, 20000))                                  # through moved vertices: the watertight intersector's edge and vertex rules
        a, b = c.trace_rays(edge), o.trace_rays(edge)
        assert hits_bit_equal(a, b).all() and (b["t"] >= 0).mean() > 0.9
        rays[:, 7] = rng.uniform(0.5, 40.0, len(rays)).astype(np.float32)                           # bounded segments, any-hit (the city's alpha-tested canopies)
        assert np.array_equal(c.trace_rays(rays, any_hit=True)["t"] >= 0, o.trace_rays(rays, any_hit=True)["t"] >= 0)
        c.close()
    fresh.close(); o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("which", ["cornell", "city"])
def test_collapsed_instance_is_never_hit(product, oracle, cornell, small_city, strict, which):
    """Scale 0 on every axis is how hosts hide an instance: its triangles and every node over them collapse to a point (zero-extent boxes)."""
    from test_gpu_parity import hits_bit_equal, random_rays
    scene = (cornell if which == "cornell" else small_city)[0]
    hidden = 2 if which == "cornell" else 5
    mats = mixed_motion(scene, start=2 if which == "cornell" else 0); mats[hidden] = about(np.zeros((3, 3)), instance_centres(scene)[hidden])
    (lo, hi), origin = _box_and_origin(which)
    rng = np.random.default_rng(22)
    c = product.Context(strict=strict); c.upload_scene(scene)
    rays = random_rays(rng, 300000, lo, hi)
    assert (c.trace_rays(rays)["inst"] == hidden).mean() > 0.001                                  # the instance is in view before
    c.update_instance_transforms(mats)
    nodes, box = c.scene_raw(0), c.scene_raw(6)
    assert np.isfinite(box).all() and np.isfinite(nodes[:, 0:3].view(np.float32)).all()
    o = oracle.Oracle(moved_scene(scene, mats))
    a, b = c.trace_rays(rays), o.trace_rays(rays)
    assert hits_bit_equal(a, b).all() and not (a["inst"][a["t"] >= 0] == hidden).any()
    edge = _rays_at(origin, _targets(scene, mats, rng, 20000))
    a, b = c.trace_rays(edge), o.trace_rays(edge)
    assert hits_bit_equal(a, b).all() and not (a["inst"][a["t"] >= 0] == hidden).any()
    rays[:, 7] = rng.uniform(0.5, 40.0, len(rays)).astype(np.float32)
    assert np.array_equal(c.trace_rays(rays, any_hit=True)["t"] >= 0, o.trace_rays(rays, any_hit=True)["t"] >= 0)
    c.close(); o.close()


def _frame_pair(product, oracle, scene, moved, consts, strict):
    c = product.Context(max_sub_samples_per_launch=4, strict=strict); c.upload_scene(scene); c.set_constants(consts)
    c.update_instance_transforms(np.stack([np.float32(moved.instances[i].transform[:]).reshape(3, 4) for i in range(moved.desc.instanceCount)]))
    c.reset_accumulation(); c.path_trace(0, 1); img = c.readback_accumulated(); st = c.stats(); c.close()
    o = oracle.Oracle(moved); o.set_constants(consts); acc, _, _, _, ost = o.render(0, 1); o.close()
    return img, st, acc, ost


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_cornell_frame_after_refit_equals_the_oracle(product, oracle, cornell, strict):
    """Shading of a refitted scene: the new instance matrices reach the hit points and the normals (xfVector of a rotated, mirrored, non-uniformly scaled instance).  The lamp stays
    where it was uploaded (its light-table entries are not re-baked).  Bars of test_gpu_parity.test_cornell_c1_image_parity."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = cornell
    cen = instance_centres(scene)
    room = about(rotation((1, 3, -2), 0.03), cen[0], (0.05, 0.0, 0.1))
    boxes = about(rotation((1, 2, 0.5), 0.4) @ np.diag([-1.1, 0.8, 1.0]), cen[2], (0.1, 0.2, 0.0))
    moved = moved_scene(scene, [room, sb.identity34(), boxes])
    consts = sb.make_constants(256, 256, cam, bounce_count=2, diffuse_bounce_count=2)
    img, st, acc, ost = _frame_pair(product, oracle, scene, moved, consts, strict)
    img0, _, _, _ = _frame_pair(product, oracle, scene, scene, consts, strict)
    assert (np.abs(img - img0).max(-1) > 0).mean() > 0.2                                          # the frame did change
    d = np.abs(img[..., :3] - acc[..., :3])
    if strict:
        assert st.scatterRays == ost.scatterRays and st.shadowRays == ost.shadowRays
        assert (d.max(-1) == 0).mean() > 0.995
        assert d.max() < 2e-2 and per_pixel_l2(img, acc) < 1e-7
    else:
        assert abs(int(st.scatterRays) - int(ost.scatterRays)) <= 1e-3 * ost.scatterRays and abs(int(st.shadowRays) - int(ost.shadowRays)) <= 1e-3 * ost.shadowRays
        rel = d / (np.abs(acc[..., :3]) + 1e-2)
        assert (rel.max(-1) < 2e-2).mean() > 0.998 and per_pixel_l2(img, acc) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_city_frame_after_refit_equals_the_oracle(product, oracle, small_city, strict):
    """The city with every instance but the emissive lamps (the last instance) on its own matrix.  1-spp bars of test_gpu_parity.test_city_image_parity_and_accumulation."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = small_city
    n = scene.desc.instanceCount
    moved = moved_scene(scene, mixed_motion(scene, fixed=(n - 1,)))
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0)
    img, st, acc, ost = _frame_pair(product, oracle, scene, moved, consts, strict)
    assert abs(int(st.scatterRays) - int(ost.scatterRays)) < 2e-3 * ost.scatterRays
    rel = np.abs(img[..., :3] - acc[..., :3]) / (np.abs(acc[..., :3]) + 1e-2)
    assert (rel.max(-1) < 5e-2).mean() > 0.995
    assert per_pixel_l2(img, acc) < 1e-3


@pytest.mark.gpu
def test_moving_the_lamp_keeps_the_uploaded_light_table(product, cornell):
    """Emissive triangles are baked into the light table at upload and not re-baked after a refit (DESIGN §2 row f4): moving the lamp instance moves what rays hit, not the lights."""
    from rtxpt_b200 import scene_builder as sb
    scene, cam = cornell
    ident = sb.identity34()
    c = product.Context(strict=True); c.upload_scene(scene); c.set_constants(sb.make_constants(256, 256, cam, bounce_count=2, diffuse_bounce_count=2))
    lights0 = c.lights()
    rays = _rays(200000, np.random.default_rng(23)); h0 = c.trace_rays(rays)
    c.update_instance_transforms(np.stack([ident, about(rotation((0, 1, 0), 0.5), instance_centres(scene)[1], (0.4, -0.8, 0.3)), ident]))
    h1 = c.trace_rays(rays)
    assert ((h0["inst"] == 1) != (h1["inst"] == 1)).sum() > 100
    assert all(np.array_equal(a, b) for a, b in zip(c.lights(), lights0))
    c.close()
