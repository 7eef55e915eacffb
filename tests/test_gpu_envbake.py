"""GPU: rtxpt_b200_bake_env_map (envbake_kernels.cu) against the oracle.  Tolerances marked "measured" come from GPU runs of these tests.  The kernels are built with IEEE arithmetic in both libraries;
atan2 / acos / pow / cos come from libdevice, so texels agree within a few fp16 steps rather than bit for bit - the tolerance below is a first estimate."""
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


@unverified
def test_bake_matches_oracle_and_feeds_the_path_tracer(product, oracle):
    from rtxpt_b200 import scene_builder as sb, scenes
    from test_envbake import _bake
    rng = np.random.default_rng(4)
    eq = rng.gamma(2.0, 0.5, (128, 256, 4)).astype(np.float32)
    d = np.float32([0.2, -0.9, 0.4]); d /= np.linalg.norm(d)
    lights = [((1.0, 0.9, 0.7), 20.0, tuple(d), 0.05)]
    scene, cam = scenes.cornell_box(64, 64)
    c = product.Context(); c.upload_scene(scene)
    got = c.bake_env_map(128, eq, scale_color=(1.0, 0.8, 0.6), lights=lights)
    want = _bake(oracle.lib(), "oracle_bake_env_map", 128, eq, (1.0, 0.8, 0.6), lights)
    assert len(got) == len(want) == 8
    for m, (x, y) in enumerate(zip(got, want)):
        assert np.isclose(x, y, rtol=4e-3, atol=1e-4).mean() > 0.999, (m, np.abs(x - y).max())
        assert np.array_equal(x, x.astype(np.float16).astype(np.float32))
    assert np.array_equal(c.bake_env_map(128, eq, scale_color=(1.0, 0.8, 0.6), lights=lights)[0], got[0])        # deterministic
    c.close()
