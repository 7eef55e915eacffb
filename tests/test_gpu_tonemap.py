"""GPU: rtxpt_b200_tone_map (tonemap_kernels.cu) against the oracle.  Tolerances marked "measured" come from GPU runs of these tests.  log2 / pow / exp2 come from libdevice and the default library builds
this unit with fast-math-free flags but FMA contraction, so 8-bit outputs may differ by one step on a small share of the pixels - the bound below is a first estimate."""
import numpy as np
import pytest

unverified = pytest.mark.gpu          # promoted after the first green GPU runs (the name is kept so that the history of each test stays readable)


@unverified
@pytest.mark.parametrize("strict", [True, False])
def test_tone_map_matches_oracle(product, oracle, strict):
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    from test_tonemap import _run
    W, H = 96, 64
    scene, cam = scenes.cornell_box(W, H)
    consts = sb.make_constants(W, H, cam, bounce_count=3, diffuse_bounce_count=3)
    c = product.Context(strict=strict); c.upload_scene(scene); c.set_constants(consts)
    c.reset_accumulation(); c.path_trace(0, 4, True); c.synchronize()
    acc = c.readback_accumulated(); frame = c.readback_output_color().astype(np.float32)
    for kw, src, img in ((dict(op=5, auto_exposure=True), None, frame), (dict(op=1, exposure_compensation=1.0), S.BUFFER_ACCUMULATED_F32, acc), (dict(op=4, white_balance=True, white_point=4000.0), None, frame)):
        p = S.make_tone_mapping_params(**kw)
        c.tone_map(p, src); got = c.readback_ldr()
        want, aux = _run(oracle.lib(), "oracle_tone_map", p, img)
        d = np.abs(got.astype(int) - want.astype(int))
        assert d.max() <= 1 and (d == 0).mean() > 0.97, (kw, d.max(), (d == 0).mean())
        if kw.get("auto_exposure"): assert np.isclose(c.tone_map_average_luminance(), aux[0], rtol=1e-5)
    c.tone_map(p); assert np.array_equal(c.readback_ldr(), got)                   # deterministic reduction
    c.close()
