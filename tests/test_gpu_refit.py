"""GPU: rtxpt_b200_update_instance_transforms (refit_kernels.cu).  Tolerances marked "measured" come from GPU runs of these tests.  The refit re-transforms the leaf triangles with the arithmetic of the
scene upload, so a refitted context must trace exactly like a context (and an oracle) that was given the moved scene from the start."""
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
