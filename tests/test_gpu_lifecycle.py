"""GPU: a context returns every CUDA resource it took (device arrays, streams, events, textures, the pinned counter block) when it is closed, whichever pools it went
through and whichever calls were refused on the way.  rtxpt_b200_debug_live_resources counts what one library holds across the process."""
import ctypes as C
import gc
import numpy as np
import pytest
from bsdf_records import make_records


def _live(L):
    n = C.c_uint64()
    assert L.rtxpt_b200_debug_live_resources(C.byref(n)) == 0
    return n.value


@pytest.mark.gpu
@pytest.mark.parametrize("strict", [False, True])
def test_closed_contexts_hold_no_resources(product, monkeypatch, strict):
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    W, H = 160, 96
    scene, cam = scenes.city_block(target_triangles=60000, width=W, height=H, texture_size=64, n_textures=4, n_materials=64)
    consts = sb.make_constants(W, H, cam, bounce_count=3, diffuse_bounce_count=2)
    d = scene.desc; rng = np.random.default_rng(5)
    L = product.load(strict)
    gc.collect(); gc.disable()          # contexts earlier tests left to the collector must not be destroyed inside the counted window
    try:
        before = _live(L)
        monkeypatch.setenv("RTXPT_LANES", "2")          # read at creation: path_trace splits each launch of two sub-samples over two lanes
        c = product.Context(max_sub_samples_per_launch=2, strict=strict)
        timed = product.Context(max_sub_samples_per_launch=2, flags=S.CFG_TIME_KERNELS, strict=strict)
        for ctx in (c, timed):
            ctx.upload_scene(scene); held = _live(L)
            ctx.upload_scene(scene); assert _live(L) == held         # the second upload frees the first scene
            ctx.set_constants(consts)
        assert c.opacity_mask_stats().triangles > 0               # alpha-tested foliage has opacity masks
        c.set_view(sb.world_to_clip(cam))
        c.path_trace(0, 4); timed.path_trace(0, 4)
        assert timed.stats().msTraceClosest > 0                     # per-kernel events from the pool
        # realtime frame, denoiser inputs and ReBLUR pools, tone mapping
        c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=3, sub_samples=1))
        c.path_trace_realtime(False); c.denoise_realtime(sb.make_denoiser_constants(cam), sb.make_reblur_frame(cam, cam))
        c.tone_map(S.make_tone_mapping_params(op=5, auto_exposure=True))
        # NEE-AT feedback state, dropped by neeat_reset and made again
        consts.NEEATFeedback = 1; c.set_constants(consts)
        c.neeat_update_begin(); c.neeat_update_end(); c.neeat_reset(); c.neeat_update_begin(); c.neeat_update_end()
        consts.NEEATFeedback = 0; c.set_constants(consts)
        # a skin on a facade without a previous-position stream (registration grows the previous-position table), then a refit
        inst = d.instances[0]; g = d.geometries[inst.firstGeometryIndex]
        assert g.prevPositionOffset == 0xFFFFFFFF
        pos = np.ctypeslib.as_array((C.c_float * (3 * g.numVertices)).from_address(d.buffers[g.vertexBufferIndex].data + g.positionOffset)).reshape(-1, 3).copy()
        ji = np.zeros((len(pos), 4), np.uint16); jw = np.zeros((len(pos), 4), np.float32); jw[:, 0] = 1
        sid = c.skin_register(0, 0, pos, ji, jw); c.skin_update(sid, np.eye(4, dtype=np.float32)[None])
        c.update_instance_transforms(np.stack([np.ctypeslib.as_array(d.instances[i].transform) for i in range(d.instanceCount)]))
        # temporary device arrays of the one-shot calls
        c.bake_env_map(16, lights=[((1.0, 1.0, 1.0), 5.0, (0.0, -1.0, 0.0), 0.05)])
        rays = np.zeros((2000, 8), np.float32); rays[:, 0:3] = (0.0, 20.0, 0.0); rays[:, 4:7] = rng.normal(0, 1, (2000, 3)); rays[:, 7] = 1e30
        rays[:, 4:7] /= np.linalg.norm(rays[:, 4:7], axis=1, keepdims=True)
        assert (c.trace_rays(rays)["t"] >= 0).any()
        c.debug_bsdf(make_records(rng, 1000)); c.debug_rng(rng.integers(0, 1 << 16, (1000, 4)))
        # refused on the host, before or after the context allocated anything
        with pytest.raises(product.RtxptError): c.skin_register(0, 0, pos[:-1], ji[:-1], jw[:-1])                  # bind pose shorter than the geometry
        with pytest.raises(product.RtxptError): c.skin_update(sid + 1, np.eye(4, dtype=np.float32)[None])           # unknown skin
        with pytest.raises(product.RtxptError): c.update_instance_transforms(np.zeros((1, 12), np.float32))        # wrong instance count
        with pytest.raises(product.RtxptError): c.bake_env_map(24)                                                 # not a power of two
        with pytest.raises(product.RtxptError): c.denoiser_prepare_inputs(3, True, sb.make_denoiser_constants(cam))   # no such plane
        with pytest.raises(product.RtxptError): product.Context(tile_rank=2, tile_world=2, strict=strict)          # bad tile partition
        c.synchronize(); assert _live(L) > before
        c.close(); timed.close()
        assert _live(L) == before
    finally:
        gc.enable()
