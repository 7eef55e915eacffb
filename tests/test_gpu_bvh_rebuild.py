"""GPU: rtxpt_b200_rebuild_bvh (bvh_build_kernels.cu).  Both libraries link the IEEE build of the rebuild kernels, so the device tree must equal the host build of the same bodies
(tests/emu: emu_build_bvh) word for word; a rebuilt tree must trace exactly like the oracle and like a fresh upload of the moved scene, refit like an uploaded one, and bring the SAH
expectations of a far-moved scene back to those of a fresh host build."""
import ctypes as C
import numpy as np
import pytest
from test_gpu_refit import mixed_motion, moved_scene, strided_city, sm_count, _rays_at, _targets, _box_and_origin  # noqa: F401  (strided_city: fixture)
from test_bvh_rebuild import emu_build, check_layout, chain_soup


def soup_scene(soup):
    """One instance, one geometry: the (n, 9) soup as it is, gid = soup index."""
    from rtxpt_b200 import scene_builder as sb
    b = sb.SceneBuilder(); m = b.add_material(sb.Material())
    v = np.ascontiguousarray(soup, np.float32).reshape(-1, 3)
    b.add_instance(b.add_mesh([dict(positions=v, indices=np.arange(len(v), dtype=np.uint32).reshape(-1, 3), normals=np.tile(np.float32([0, 0, 1]), (len(v), 1)), material=m)]), sb.identity34())
    return b.build()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_rebuild_equals_the_host_build_where_the_launch_strides(product, strided_city, strict):
    scene = strided_city
    c = product.Context(strict=strict); c.upload_scene(scene)
    c.update_instance_transforms(mixed_motion(scene, far=True))
    tris0 = c.scene_raw(1)
    assert len(tris0) > sm_count() * 8 * 256                                                        # every grid-stride loop over triangles takes more than one pass
    st, want_n, want_t, want_b, want_l, it = emu_build(tris0)
    assert st == 0
    for _ in range(2):                                                                               # the same inputs twice: the same words
        c.rebuild_bvh()
        n, t, l = c.scene_raw(0), c.scene_raw(1), c.scene_raw(5)
        assert np.array_equal(l, want_l) and np.array_equal(n, want_n) and np.array_equal(t, want_t)
        assert len(c.scene_raw(6)) == 0
    check_layout(n, t, l, tris0)
    print(f"\n{len(t)} triangles: {len(n)} nodes in {len(l) - 1} levels, {it} PLOC iterations, rebuild {c.bvh_stats().buildSeconds * 1e3:.2f} ms")
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
@pytest.mark.parametrize("which", ["cornell", "city"])
def test_rebuilt_tree_traces_like_the_oracle(product, oracle, cornell, small_city, monkeypatch, strict, which):
    import host_build_lib as emu
    from test_gpu_parity import hits_bit_equal, random_rays
    from test_refit import _refit
    scene = (cornell if which == "cornell" else small_city)[0]
    mats = mixed_motion(scene, far=True, start=2 if which == "cornell" else 0)
    moved = moved_scene(scene, mats)
    o = oracle.Oracle(moved); fresh = product.Context(strict=strict); fresh.upload_scene(moved)
    (lo, hi), origin = _box_and_origin(which)
    for smem in (None, "200"):                                                                      # 200: the top of the tree is staged in shared memory (read at context creation)
        if smem: monkeypatch.setenv("RTXPT_SMEM_NODES", smem)
        rng = np.random.default_rng(31)
        c = product.Context(strict=strict); c.upload_scene(scene)
        c.update_instance_transforms(mats); c.rebuild_bvh()
        rays = random_rays(rng, 300000, lo, hi)
        a, b = c.trace_rays(rays), o.trace_rays(rays)
        assert hits_bit_equal(a, b).all() and hits_bit_equal(a, fresh.trace_rays(rays)).all()
        edge = _rays_at(origin, _targets(scene, mats, rng, 20000))
        a, b = c.trace_rays(edge), o.trace_rays(edge)
        assert hits_bit_equal(a, b).all() and (b["t"] >= 0).mean() > 0.5
        seg = rays.copy(); seg[:, 7] = rng.uniform(0.5, 40.0, len(seg)).astype(np.float32)     # bounded segments, any-hit (the city's alpha-tested canopies)
        assert np.array_equal(c.trace_rays(seg, any_hit=True)["t"] >= 0, o.trace_rays(seg, any_hit=True)["t"] >= 0)
        # an identity refit returns the rebuilt tree word for word; a further motion, refitted, still traces like the oracle
        nodes, tris, levels = c.scene_raw(0), c.scene_raw(1), c.scene_raw(5)
        c.update_instance_transforms(mats)
        assert np.array_equal(c.scene_raw(0), nodes) and np.array_equal(c.scene_raw(1), tris)
        _, _, want_b = _refit(emu, nodes, tris, c.scene_raw(2), mats, levels)
        assert np.array_equal(c.scene_raw(6).view(np.uint32), want_b.view(np.uint32))
        mats2 = mixed_motion(scene, start=3)
        c.update_instance_transforms(mats2)
        o2 = oracle.Oracle(moved_scene(scene, mats2))
        assert hits_bit_equal(c.trace_rays(rays), o2.trace_rays(rays)).all()
        o2.close(); c.close()
    fresh.close(); o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_city_frame_after_rebuild_equals_a_fresh_upload(product, oracle, small_city, strict):
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    scene, cam = small_city
    n = scene.desc.instanceCount
    mats = mixed_motion(scene, fixed=(n - 1,)); moved = moved_scene(scene, mats)
    W, H = cam.ViewportSize[0], cam.ViewportSize[1]
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0)
    c = product.Context(max_sub_samples_per_launch=4, strict=strict); c.upload_scene(scene); c.set_constants(consts)
    c.update_instance_transforms(mats); c.rebuild_bvh()
    c.reset_accumulation(); c.path_trace(0, 1); img = c.readback_accumulated(); st = c.stats(); c.close()
    f = product.Context(max_sub_samples_per_launch=4, strict=strict); f.upload_scene(moved); f.set_constants(consts)
    f.update_instance_transforms(mats)                                                              # the same previous-frame matrices as the rebuilt context (motion vectors)
    f.reset_accumulation(); f.path_trace(0, 1); ref = f.readback_accumulated(); fst = f.stats(); f.close()
    assert st.scatterRays == fst.scatterRays and st.shadowRays == fst.shadowRays
    same = (img == ref).all(-1).mean()
    print(f"\n{100 * same:.4f} % of pixels bit-identical to a fresh upload")
    assert same >= 0.9999
    o = oracle.Oracle(moved); o.set_constants(consts); acc, _, _, _, ost = o.render(0, 1); o.close()
    assert per_pixel_l2(img, acc) < 1e-3


@pytest.mark.gpu
def test_skinned_then_rebuilt_traces_like_the_refit(product, cornell):
    """skin_update -> update_instance_transforms -> rebuild_bvh traces like the same updates refitted, which tests/test_gpu_skinning.py holds to the oracle."""
    from test_gpu_parity import hits_bit_equal, random_rays
    from test_gpu_refit import instance_centres, about, rotation
    from rtxpt_b200 import scene_builder as sb
    scene = cornell[0]
    inst = scene.instances[2]; g = scene.geometries[inst.firstGeometryIndex]
    pos = np.ctypeslib.as_array((C.c_float * (g.numVertices * 3)).from_address(scene.buffers[g.vertexBufferIndex].data + g.positionOffset)).reshape(-1, 3).copy()
    joints = np.zeros((len(pos), 4), np.uint16); joints[:, 1] = 1; w = np.zeros((len(pos), 4), np.float32); w[:, 0] = 0.5; w[:, 1] = 0.5
    cen = pos.mean(0); J0 = np.eye(4, dtype=np.float32); J1 = np.eye(4, dtype=np.float32)
    J1[:3, :3] = rotation((0, 1, 0), 0.6).T; J1[3, :3] = cen - cen @ rotation((0, 1, 0), 0.6).T + np.float32([0.3, 0.0, 0.2])
    c = product.Context(strict=True); c.upload_scene(scene)
    sid = c.skin_register(2, 0, pos, joints, w)
    c.skin_update(sid, np.stack([J0, J1]))
    ident = np.stack([np.float32(scene.instances[i].transform[:]).reshape(3, 4) for i in range(scene.desc.instanceCount)])
    c.update_instance_transforms(ident); c.rebuild_bvh()
    rays = random_rays(np.random.default_rng(33), 200000, [0.1, 0.1, -4.0], [5.4, 5.4, 5.4])
    a = c.trace_rays(rays)
    r = product.Context(strict=True); r.upload_scene(scene); sid2 = r.skin_register(2, 0, pos, joints, w); r.skin_update(sid2, np.stack([J0, J1])); r.update_instance_transforms(ident)
    assert hits_bit_equal(a, r.trace_rays(rays)).all()
    assert (a["inst"] == 2).mean() > 0.01
    r.close(); c.close()


@pytest.mark.gpu
def test_quality_comes_back_after_a_rebuild(product, small_city):
    scene = small_city[0]
    mats = mixed_motion(scene, far=True)
    c = product.Context(); c.upload_scene(scene)
    c.update_instance_transforms(mats); refit = c.bvh_stats()
    c.rebuild_bvh(); rebuilt = c.bvh_stats()
    f = product.Context(); f.upload_scene(moved_scene(scene, mats)); fresh = f.bvh_stats(); f.close()
    print(f"\nE[node visits] / E[triangle tests]: refit only {refit.expectedNodeVisits:.2f} / {refit.expectedTriangleTests:.2f}, rebuilt {rebuilt.expectedNodeVisits:.2f} / "
          f"{rebuilt.expectedTriangleTests:.2f}, fresh upload {fresh.expectedNodeVisits:.2f} / {fresh.expectedTriangleTests:.2f}; refit-only / fresh: "
          f"{refit.expectedNodeVisits / fresh.expectedNodeVisits:.2f}x / {refit.expectedTriangleTests / fresh.expectedTriangleTests:.2f}x; rebuild {rebuilt.buildSeconds * 1e3:.2f} ms")
    assert rebuilt.expectedNodeVisits <= 1.25 * fresh.expectedNodeVisits and rebuilt.expectedTriangleTests <= 1.2 * fresh.expectedTriangleTests
    assert refit.expectedNodeVisits > rebuilt.expectedNodeVisits
    assert rebuilt.nodeCount == len(c.scene_raw(0)) and rebuilt.maxDepth == len(c.scene_raw(5)) - 1 and rebuilt.triangleReferenceCount == len(c.scene_raw(1))
    c.close()


@pytest.mark.gpu
def test_host_tree_stats_equal_the_inspection_hook(product):
    """bvh_stats() of an uploaded soup equals rtxpt_b200_debug_bvh_stats on the same soup (one SAH function, bvh_builder.cpp)."""
    from rtxpt_b200 import scene_builder as sb
    from test_refit import _soup
    soup, _ = _soup(5000, np.random.default_rng(44))
    c = product.Context(); c.upload_scene(soup_scene(soup))
    got, want = c.bvh_stats(), product.bvh_stats(soup)
    for k in ("nodeCount", "triangleReferenceCount", "leafCount", "maxDepth", "expectedNodeVisits", "expectedTriangleTests"):
        assert getattr(got, k) == getattr(want, k), k
    c.close()


@pytest.mark.gpu
def test_too_deep_no_scene_and_lifecycle(product):
    from rtxpt_b200 import scene_builder as sb
    from test_gpu_parity import hits_bit_equal, random_rays
    L = product.load()
    live0 = C.c_uint64(); assert L.rtxpt_b200_debug_live_resources(C.byref(live0)) == 0
    c = product.Context()
    assert L.rtxpt_b200_rebuild_bvh(c.h, None) == -5                                               # RTXPT_ERR_NO_SCENE
    soup = chain_soup()
    deep = soup_scene(soup)
    c.upload_scene(deep)
    rays = random_rays(np.random.default_rng(35), 50000, [-1, -1, -1], [300, 3e15, 3e15])
    before, nodes = c.trace_rays(rays), c.scene_raw(0)
    assert L.rtxpt_b200_rebuild_bvh(c.h, None) == -6                                               # RTXPT_ERR_UNSUPPORTED: deeper than the traversal stack
    assert np.array_equal(c.scene_raw(0), nodes) and hits_bit_equal(c.trace_rays(rays), before).all()
    c.close()
    c = product.Context(); c.upload_scene(deep)
    for _ in range(3): L.rtxpt_b200_rebuild_bvh(c.h, None)
    c.close()
    from rtxpt_b200 import scenes
    c = product.Context(); c.upload_scene(scenes.cornell_box(64, 64)[0])
    for _ in range(3): c.rebuild_bvh()
    c.close()
    live = C.c_uint64(); assert L.rtxpt_b200_debug_live_resources(C.byref(live)) == 0
    assert live.value == live0.value
