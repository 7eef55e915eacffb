"""GPU: rtxpt_b200_skin_register / rtxpt_b200_skin_update (skinning_kernels.cu) + the refit.  Tolerances marked "measured" come from GPU runs of these tests.  A context whose boxes were bent by a
two-joint skin must trace exactly like a fresh upload of the bent mesh (and like the oracle on it): the skin writes the same float positions a host-side blend produces."""
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
