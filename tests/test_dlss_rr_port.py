"""CPU: RTXPT's DLSS-RR input pass (PostProcess.hlsl DENOISER_DLSS_RR, rtxpt_b200_dlss_rr_prepare_inputs) against the reference and the oracle.  The oracle's restatement
(oracle/pt_dlss_rr.h) and the host build of the product's pixel bodies (tests/emu/dlss_rr.mk) reproduce tests/golden/dlss_rr_golden.npz - what the UNMODIFIED shader computes
(oracle/_ref/ref_kat_dlss_rr) - word for word; on whole synthetic frames the host build gives the oracle's stores word for word.  The oracle's outputs hold the pass's
properties: unit guide normals, an average albedo of at least 0.05, zero specular motion under an unchanged camera, and on a planar mirror the analytic motion of the mirrored image."""
import numpy as np
import pytest

from rtxpt_b200 import structs as S
import dlss_rr_lib as D

INVALID = 0xFFFFFFFF


def _words(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_golden_covers_the_cases():
    inp, out = D.golden()
    assert set(np.unique(inp[:, 0])) == {1, 2, 3}
    branches = inp[:, 2:5]
    assert (branches == INVALID).any() and (branches != INVALID).all(1).any() and (branches == INVALID).all(1).any()
    scene_length = inp[:, 6 + 7: 66: 20].view(np.float32)
    assert np.isinf(scene_length).any()
    assert set(np.unique(inp[:, 1].view(np.float32))) == {0.5, 4096.0}
    spec_hit_t = inp[:, 68].view(np.float32)
    t = np.float32(1e-3)
    for v in (t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))):
        assert (spec_hit_t == v).any()
    assert ((inp[:, 66] == 0) & (inp[:, 67] & 0xFFFF == 0)).any()            # zero stable radiance
    static = (inp[:, 70:86] == inp[:, 86:102]).all(1)
    assert static.any() and (~static).any()
    guide = np.stack([(inp[:, 69] & 0xFFFF).astype(np.uint16), (inp[:, 69] >> 16).astype(np.uint16)], -1)
    taken = (out[:, 13:15].astype(np.float16).view(np.uint16) != guide).any(1)
    assert taken.sum() > 50 and (~taken).sum() > 50                 # both sides of the specular-motion test
    assert (out[:, 12] < 0.25).any() and (out[:, 12] > 0.25).any()
    avg = lambda a: ((a[:, 0] + a[:, 1]) + a[:, 2]) / np.float32(3)
    diff, spec = out[:, 3:6], out[:, 6:9]
    assert ((avg(diff) < 0.05) & (avg(diff + spec) >= 0.05)).sum() > 20      # a dark diffuse guide the specular one alone keeps above the 0.05 floor


@pytest.mark.parametrize("which", ["oracle", "emu"])
def test_reproduces_reference_golden(which):
    inp, out = D.golden()
    got = D.records(which, inp)
    bad = np.nonzero((_words(got) != _words(out)).any(1))[0]
    assert len(bad) == 0, (which, len(bad), bad[:8], got[bad[:2]], out[bad[:2]])


def test_oracle_properties_on_golden():
    inp, _ = D.golden()
    out = D.records("oracle", inp)
    n = out[:, 9:12].astype(np.float64)
    assert np.abs(np.linalg.norm(n, axis=1) - 1.0).max() < 1e-6
    albedo = out[:, 3:6] + out[:, 6:9]
    assert (((albedo[:, 0] + albedo[:, 1]) + albedo[:, 2]) / np.float32(3) >= np.float32(0.05) * (1 - 1e-6)).all()


def _frame_from_records(inp, W, H, active, rng):
    """A synthetic W x H frame whose pixels take golden records' planes, header, radiance, hit distance and motion; one camera and plane count per frame."""
    line = (W + 7) // 8 * 8; plane_stride = line * ((H + 7) // 8 * 8)
    planes = np.zeros((3 * plane_stride, 20), np.uint32)
    header = np.zeros((4, H, W), np.uint32); sr = np.zeros((H, W, 2), np.uint32); mv = np.zeros((H, W, 2), np.uint32); sh = np.zeros((H, W), np.uint32)
    pick = rng.integers(0, len(inp), W * H)

    def morton(x, y):
        r = 0
        for b in range(3): r |= ((x >> b) & 1) << (2 * b) | ((y >> b) & 1) << (2 * b + 1)
        return r
    for k, (y, x) in enumerate(np.ndindex(H, W)):
        r = inp[pick[k]]
        header[:, y, x] = r[2:6]
        for p in range(3):
            planes[(x - x % 8) * 8 + (y - y % 8) * line + morton(x % 8, y % 8) + p * plane_stride] = r[6 + 20 * p: 26 + 20 * p]
        sr[y, x] = r[66:68]; sh[y, x] = r[68]; mv[y, x, 0] = r[69]
    rt = S.RealtimeConstants(); rt.activeStablePlaneCount = active; rt.subSampleCount = 1
    r = inp[pick[0]]
    rt.matWorldToClipNoOffset[:] = r[70:86].view(np.float32).tolist(); rt.prevMatWorldToClipNoOffset[:] = r[86:102].view(np.float32).tolist()
    rt.clipToWindowScale[:] = r[102:104].view(np.float32).tolist()
    bufs = dict(planes=planes, header=header, stable_radiance=sr.view(np.float16).reshape(H, W, 4),
                motion=mv.view(np.float16).reshape(H, W, 4), spec_hit_t=sh.view(np.float32))
    return rt, bufs


@pytest.mark.parametrize("W,H,active,clamp", [(37, 29, 3, 4096.0), (16, 9, 2, 0.5), (1, 13, 1, 4096.0), (24, 24, 3, 0.5)])
def test_host_build_matches_oracle_frame(W, H, active, clamp):
    inp, _ = D.golden()
    rt, bufs = _frame_from_records(inp, W, H, active, np.random.default_rng(W * 1000 + H))
    bad = D.mismatches(D.frame("oracle", rt, bufs, clamp), D.frame("emu", rt, bufs, clamp))
    assert not any(bad.values()), bad


def _mirror_records(static, count=400, seed=5):
    """One active plane: a planar mirror y = 0 seen from a camera, rough 0.1, a reflection hit at distance t; the guide motion is a sentinel."""
    g = D.generator(); rng = np.random.default_rng(seed)
    eye = np.array([0.3, 2.0, -6.0]); cur = g.world_to_clip(eye, [0, 0, 0])
    prev = cur if static else g.world_to_clip(eye + [0.2, -0.1, 0.15], [0.05, 0.0, 0.1])
    recs = np.zeros((count, 104), np.uint32); hits = []
    for i in range(count):
        P = np.array([rng.uniform(-3, 3), 0.0, rng.uniform(-2, 4)]); t = rng.uniform(0.5, 10)
        d = P - eye; length = np.linalg.norm(d); d /= length
        r = recs[i]; r[0] = 1; r[1] = np.float32(4096).view(np.uint32); r[2:5] = [1, INVALID, INVALID]; r[5] = 0
        s = r[6:26]
        s[0:3] = eye.astype(np.float32).view(np.uint32); s[4:7] = d.astype(np.float32).view(np.uint32); s[7] = np.float32(length).view(np.uint32)
        s[8:11] = g.pack2(np.full(3, 0.8), np.zeros(3)); s[11] = (1 << 16) | g.f16(0.1); s[12:15] = g.pack2(np.full(3, 0.5), np.full(3, 0.5))
        s[15] = g.oct_word(np.array([0.0, 1.0, 0.0]))
        r[68] = np.float32(t).view(np.uint32); r[69] = g.f16(7.0) | (g.f16(-3.0) << 16)
        r[70:86] = cur.reshape(-1).view(np.uint32); r[86:102] = prev.reshape(-1).view(np.uint32); r[102:104] = np.float32([0.5 * g.W, -0.5 * g.H]).view(np.uint32)
        hits.append((eye.astype(np.float32).astype(np.float64) + d.astype(np.float32) * np.float32(length), d, t))
    return recs, hits, cur.astype(np.float64), prev.astype(np.float64)


def test_specular_motion_zero_under_unchanged_camera():
    recs, _, _, _ = _mirror_records(static=True)
    out = D.records("oracle", recs)
    assert (out[:, 13:15] == 0).all()
    inp, gout = D.golden()
    static = (inp[:, 70:86] == inp[:, 86:102]).all(1)
    guide = np.stack([(inp[:, 69] & 0xFFFF).astype(np.uint16).view(np.float16), (inp[:, 69] >> 16).astype(np.uint16).view(np.float16)], -1).astype(np.float32)
    mv = gout[static, 13:15]
    assert ((mv == 0).all(1) | (mv == guide[static]).all(1) | np.isnan(mv).any(1)).all()     # NaN: a sky plane 0 has no hit point


def test_specular_motion_on_planar_mirror_is_image_motion():
    recs, hits, cur, prev = _mirror_records(static=False)
    out = D.records("oracle", recs)
    for (P, d, t), mv in zip(hits, out[:, 13:15]):
        image = P + d * t                     # the reflection hit mirrored behind y = 0 lies on the camera ray, t beyond the mirror
        def ndc(M):
            c = np.append(image, 1.0) @ M
            return c[:2] / c[3]
        expect = (ndc(prev) - ndc(cur)) * np.array([0.5 * 1920, -0.5 * 1080])
        assert np.abs(mv - expect).max() < 2e-3 * max(1.0, np.abs(expect).max()), (mv, expect)
        assert np.abs(expect).max() > 1e-2


def test_unpack_r11g11b10():
    from rtxpt_b200 import lib
    v = np.array([0.05, 0.5, 1.0], np.float32)
    h = v.astype(np.float16).view(np.uint16).astype(np.uint32)
    w = ((h[0] + 8) >> 4) & 0x7FF | (((h[1] + 8) << 7) & 0x3FF800) | (((h[2] + 16) << 17) & 0xFFC00000)
    assert np.allclose(lib.unpack_r11g11b10(np.uint32(w)), v, rtol=1 / 32)
