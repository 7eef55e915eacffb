"""GPU: RTXPT's DLSS-RR input pass (rtxpt_b200_dlss_rr_prepare_inputs, PostProcess.hlsl DENOISER_DLSS_RR) on real realtime frames, against the oracle (oracle/pt_dlss_rr.h) fed the
context's own realtime buffers: the strict (IEEE) build gives the oracle's stores in every word of all five targets on every pixel; in the default build (FMA contraction,
approximate division and square root) colour, albedos and normals + roughness stay within FAST_ULPS format ulps on every pixel, and the specular motion vectors within
FAST_MOTION_PX / FAST_MOTION_REL on all but FAST_MOTION_SHARE of the pixels (measured on an H100: see the bars below).  The pass writes nothing else, copies the motion-vector guide
where the specular motion test fails, splits over a tile partition like every per-pixel pass, and refuses what it cannot run."""
import numpy as np
import pytest

from rtxpt_b200 import structs as S
import dlss_rr_lib as D

STRICT = pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
RR = [S.BUFFER_OUTPUT_COLOR_F16, S.BUFFER_RR_DIFFUSE_ALBEDO_R11G11B10, S.BUFFER_RR_SPECULAR_ALBEDO_R11G11B10, S.BUFFER_RR_NORMALS_ROUGHNESS_F16, S.BUFFER_RR_SPECULAR_MOTION_VECTORS_F16]
# default build, per target: the largest difference in format ulps (fp16 ulps; R11G11B10: units of the 6 / 5-bit mantissas), on every pixel.  Specular motion vectors are held in
# pixels instead, on all but FAST_MOTION_SHARE of the pixels: under an unchanged camera the strict build's vector is exactly 0 and the default build's a contraction residue, thousands
# of fp16 ulps from 0 but far below a pixel, and the test that selects the specular vector (mixed roughness < 0.25) can come out the other way where the roughness sits on it.
# Measured on an H100 80GB HBM3 (700 W), largest over the cases: colour 0 ulps, diffuse albedo 1, specular albedo 0, normals + roughness 5; specular motion 2.4e-4 px, no pixel
# beyond its bar.
FAST_ULPS = dict(color=2, diff_albedo=2, spec_albedo=2, normals_roughness=8)
FAST_MOTION_PX, FAST_MOTION_REL = 1e-3, 2e-3
FAST_MOTION_SHARE = 2e-3
CASES = [("cornell", 96, 96, 3, 4096.0, False), ("cornell", 97, 61, 2, 0.5, True), ("cornell", 1, 64, 1, 4096.0, True), ("city", 160, 90, 3, 4096.0, True),
         ("cornell", 96, 96, 1, 0.5, False), ("cornell", 1920, 1080, 3, 4096.0, True)]


def _moved(M, offset=(0.06, -0.03, 0.04)):
    """A previous view a small camera translation away: float4(p, 1) x T x M."""
    T = np.eye(4, dtype=np.float64); T[3, :3] = offset
    return (T @ np.asarray(M, np.float64).reshape(4, 4)).astype(np.float32).reshape(16)


def _context(product, scene_name, W, H, active, moving, strict=False, **ctx_kwargs):
    from rtxpt_b200 import scene_builder as sb, scenes
    if scene_name == "city":
        from test_oracle_realtime import _opt_glass_into_decomposition
        scene, cam = scenes.city_block(target_triangles=120000, width=W, height=H, texture_size=128, n_textures=6, n_materials=64)
        _opt_glass_into_decomposition(scene)
        consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nee=True, nee_type=2)
    else:
        scene, cam = scenes.cornell_box(W, H, delta_surfaces=True)
        consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict, **ctx_kwargs); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2, active_planes=active)
    if moving: rt.prevMatWorldToClipNoOffset[:] = _moved(rt.matWorldToClipNoOffset).tolist()
    c.set_realtime(rt)
    return c, rt, scene, cam, consts


def _trace(c):
    c.path_trace_realtime(False); c.denoise_spec_hit_t(); c.synchronize()


def _ulps16(a, b):
    """fp16 distance in ulps (sign-magnitude to ordered integers); NaN pairs count 0"""
    def ordered(x):
        w = x.view(np.uint16).astype(np.int32)
        return np.where(w & 0x8000, 0x8000 - w, w)
    d = np.abs(ordered(a) - ordered(b))
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


def _ulps_r11g11b10(a, b):
    fields = [(0, 0x7FF), (11, 0x7FF), (22, 0x3FF)]
    return np.max([np.abs(((a >> s) & m).astype(np.int64) - ((b >> s) & m).astype(np.int64)) for s, m in fields], 0)


def _ulps(got, ref):
    out = {}
    for k in ("color", "normals_roughness"):
        n = 3 if k == "color" else None
        out[k] = _ulps16(got[k][..., :n], ref[k][..., :n]).max(-1)
    for k in ("diff_albedo", "spec_albedo"): out[k] = _ulps_r11g11b10(got[k], ref[k])
    return out


@pytest.mark.gpu
@STRICT
@pytest.mark.parametrize("scene_name,W,H,active,clamp,moving", CASES)
def test_matches_oracle_on_the_context_buffers(product, strict, scene_name, W, H, active, clamp, moving):
    c, rt, *_ = _context(product, scene_name, W, H, active, moving, strict)
    _trace(c)
    before = c.readback_realtime()
    c.dlss_rr_prepare_inputs(clamp); c.synchronize()
    got = c.readback_dlss_rr()
    after = c.readback_realtime()
    for k in before:                                               # every other target is what the frame left (the output colour is one of the pass's targets)
        if k != "merged": assert before[k].tobytes() == after[k].tobytes(), k
    ref = D.frame("oracle", rt, before, clamp)
    assert np.isfinite(got["color"].astype(np.float32)).all()
    if strict:
        bad = D.mismatches(got, ref)
        assert not any(bad.values()), bad
    else:
        u = _ulps(got, ref)
        print("default build vs oracle: max ulps", {k: int(v.max()) for k, v in u.items()})
        for k, v in u.items(): assert int(v.max()) <= FAST_ULPS[k], (k, int(v.max()), int((v > FAST_ULPS[k]).sum()))
        a, b = got["spec_motion"].astype(np.float32), ref["spec_motion"].astype(np.float32)
        far = (np.abs(a - b) > FAST_MOTION_PX + FAST_MOTION_REL * np.abs(b)).any(-1) & ~(np.isnan(a) & np.isnan(b)).any(-1)
        print("specular motion: largest difference %.3g px, beyond the bar on %.3g of the pixels" % (float(np.nanmax(np.abs(a - b), initial=0)), float(far.mean())))
        assert far.mean() <= FAST_MOTION_SHARE, float(far.mean())
    # where the specular motion test cannot pass (no specular hit distance), the guide's xy halves are stored as they are
    off = before["spec_hit_t"] <= 1e-3
    assert off.any()
    assert np.array_equal(got["spec_motion"].view(np.uint16)[off], before["motion"].view(np.uint16)[off][:, :2])
    unit = np.linalg.norm(got["normals_roughness"][..., :3].astype(np.float64), axis=-1)
    assert np.abs(unit - 1).max() < 2e-3
    c.close()


@pytest.mark.gpu
def test_tile_partition_reassembles_the_frame(product):
    """Two contexts owning interleaved 32 x 32 tiles run the header's recipe (trace own tiles, exchange guides, spec-hit-T filter, RR prepare own tiles, exchange the RR set):
    every rank then holds the single context's RR set bit for bit."""
    from rtxpt_b200 import realtime_mgpu as M
    W, H = 160, 128
    one, rt, *_ = _context(product, "cornell", W, H, 3, True)
    two = [_context(product, "cornell", W, H, 3, True, tile_rank=r, tile_world=2, tile_size=32)[0] for r in range(2)]
    group = M.LocalGroup(two)
    _trace(one); one.dlss_rr_prepare_inputs(); one.synchronize(); ref = one.readback_dlss_rr()
    for c in two: c.path_trace_realtime(False)
    group.exchange(M.GUIDES + [S.BUFFER_MOTION_VECTORS_F16])
    for c in two: c.denoise_spec_hit_t(); c.dlss_rr_prepare_inputs()
    group.exchange(RR)
    for c in two:
        c.synchronize(); got = c.readback_dlss_rr()
        for k in ref: assert ref[k].tobytes() == got[k].tobytes(), k
    for c in [one] + two: c.close()


@pytest.mark.gpu
def test_refusals_and_resize(product):
    from rtxpt_b200 import scene_builder as sb, scenes
    c, rt, scene, cam, consts = _context(product, "cornell", 64, 48, 3, False)
    with pytest.raises(product.RtxptError): c.dlss_rr_prepare_inputs()                     # no realtime frame yet
    for b in RR[1:]:
        with pytest.raises(product.RtxptError): c.device_ptr(b)                             # the RR targets do not exist yet
        with pytest.raises(product.RtxptError): c.exchange_bytes([b])
    _trace(c)
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(product.RtxptError): c.dlss_rr_prepare_inputs(bad)
    with pytest.raises(product.RtxptError): c.device_ptr(RR[1])                                 # a refused call allocates nothing
    c.dlss_rr_prepare_inputs(); c.synchronize()
    assert c.device_ptr(S.BUFFER_RR_NORMALS_ROUGHNESS_F16)[1] == 64 * 48 * 8 and c.exchange_bytes(RR) > 0
    # resize: the new size has no frame until one is traced; then it equals a fresh context's
    W, H = 37, 29
    scene2, cam2 = scenes.cornell_box(W, H, delta_surfaces=True)
    consts2 = sb.make_constants(W, H, cam2, bounce_count=6, diffuse_bounce_count=3)
    rt2 = sb.make_realtime_constants(W, H, cam2, bounce_count=6, sub_samples=2)
    c.set_constants(consts2); c.set_view(sb.world_to_clip(cam2)); c.set_realtime(rt2)
    with pytest.raises(product.RtxptError): c.dlss_rr_prepare_inputs()
    with pytest.raises(product.RtxptError): c.device_ptr(RR[1])
    _trace(c); c.dlss_rr_prepare_inputs(0.5); c.synchronize(); got = c.readback_dlss_rr()
    fresh = product.Context(max_sub_samples_per_launch=1); fresh.upload_scene(scene2); fresh.set_constants(consts2); fresh.set_view(sb.world_to_clip(cam2)); fresh.set_realtime(rt2)
    _trace(fresh); fresh.dlss_rr_prepare_inputs(0.5); fresh.synchronize(); ref = fresh.readback_dlss_rr()
    for k in ref: assert ref[k].shape == (H, W) + ref[k].shape[2:] and ref[k].tobytes() == got[k].tobytes(), k
    c.close(); fresh.close()
