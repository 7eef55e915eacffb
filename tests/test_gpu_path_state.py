"""GPU: the reference-mode wavefront keeps path state in ray order (wavefront.cuh): every iteration reads its rays from one state set and appends the paths
that continue to the other, while a path's radiance stays at its home index.  How the work is split and ordered must not move a single bit of the frame: pipeline
lanes, sub-samples per launch and the material sort change which ray index a path has at every bounce, so any mix-up of ray index and home index shows up as
moved radiance.  The scene has glazed shop fronts (nested dielectrics: false hits continue the path without a bounce); one run has NEE-AT feedback, whose
shadow kernel writes per-path roulette fixes and per-pixel reservoirs by home index."""
import numpy as np
import pytest

W, H, SPP = 320, 180, 4


@pytest.fixture(scope="module")
def glazed_city():
    from rtxpt_b200 import scenes, scene_builder as sb
    scene, cam = scenes.city_block(target_triangles=150000, width=W, height=H, texture_size=128, n_textures=6, n_materials=64, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nested_dielectrics=1)
    return scene, cam, consts


def _render(product, monkeypatch, glazed_city, strict, lanes=1, per_launch=SPP, flags=0, neeat=False):
    from rtxpt_b200 import scene_builder as sb, structs as S
    scene, cam, consts = glazed_city
    monkeypatch.setenv("RTXPT_LANES", str(lanes))          # read when the context is created
    c = product.Context(max_sub_samples_per_launch=per_launch, strict=strict, flags=flags | (S.CFG_EXPORT_GUIDES if neeat else 0))
    try:
        c.upload_scene(scene)
        if neeat: c.set_view(sb.world_to_clip(cam))
        frames = []
        for f in range(3):
            consts.sampleBaseIndex = f * SPP
            consts.NEEATFeedback = 1 if (neeat and f > 0) else 0        # frame 0 leaves the guides the feedback pass reprojects with
            c.set_constants(consts)
            if consts.NEEATFeedback: c.neeat_update_begin(); c.neeat_update_end()
            c.path_trace(0, SPP, True); c.synchronize()
            frames.append(c.readback_output_color().copy())
        return c.readback_accumulated(), np.stack(frames)
    finally:
        consts.NEEATFeedback = 0
        c.close()


def _same(a, b, what):
    (acc_a, col_a), (acc_b, col_b) = a, b
    assert acc_a.view(np.uint32).shape == acc_b.view(np.uint32).shape
    assert np.array_equal(acc_a.view(np.uint32), acc_b.view(np.uint32)), (what, int((acc_a != acc_b).any(-1).sum()))
    assert np.array_equal(col_a.view(np.uint16), col_b.view(np.uint16)), (what, int((col_a != col_b).any(-1).sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["fast", "strict"])
def test_frame_does_not_depend_on_how_paths_are_ordered(product, monkeypatch, glazed_city, strict):
    base = _render(product, monkeypatch, glazed_city, strict)
    acc = base[0]
    assert np.isfinite(acc).all() and acc[..., :3].mean() > 1e-3
    for lanes in (2, 4):
        _same(base, _render(product, monkeypatch, glazed_city, strict, lanes=lanes), "RTXPT_LANES=%d" % lanes)
    _same(base, _render(product, monkeypatch, glazed_city, strict, per_launch=1), "4 launches of 1 sub-sample")
    from rtxpt_b200 import structs as S
    _same(base, _render(product, monkeypatch, glazed_city, strict, flags=S.CFG_NO_MATERIAL_SORT), "no material sort")


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True], ids=["fast", "strict"])
def test_neeat_frame_does_not_depend_on_material_sort(product, monkeypatch, glazed_city, strict):
    from rtxpt_b200 import structs as S
    base = _render(product, monkeypatch, glazed_city, strict, neeat=True)
    assert np.isfinite(base[0]).all() and base[0][..., :3].mean() > 1e-3
    _same(base, _render(product, monkeypatch, glazed_city, strict, neeat=True, flags=S.CFG_NO_MATERIAL_SORT), "NEE-AT, no material sort")
