"""CPU: RTXPT's debug views (rtxpt_b200/csrc/debug_views.cuh) against the oracle's restatement (oracle/pt_debug_views.h) and the reference.  The oracle and the host build of the
header reproduce tests/golden/debug_view_golden.npz - what the UNMODIFIED ColorFromHash, GradientHeatMap, StablePlaneDebugVizColor, StablePlaneDebugVizFourWaySplitCoord and
DbgShowNormalSRGB compute (oracle/_ref/ref_kat_debug) - word for word.  The host build (tests/emu/debug_views.mk) gives the oracle's colour word for word for every first-hit view on random surfaces and for every stable-plane view on random plane buffers, at every plane index and at odd and
even image sizes.  The Python mirror of rtxpt_b200_set_debug_view's validation accepts the views the library draws and refuses the rest."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rtxpt_b200 import structs as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu():
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "debug_views.mk"], check=True)
    L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libdebug_views_emu.so"))
    L.debug_first_hit_emu.argtypes = [C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    L.debug_pixel_funcs_emu.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.debug_stable_planes_emu.argtypes = [C.c_uint32, C.c_int32] + [C.c_uint32] * 4 + [C.c_void_p] * 4
    return L


@pytest.fixture(scope="module")
def odv():
    import oracle_debug_views_lib
    oracle_debug_views_lib.build()
    return oracle_debug_views_lib


GOLDEN = os.path.join(ROOT, "tests", "golden", "debug_view_golden.npz")


def test_oracle_and_host_build_reproduce_reference_golden(emu, odv):
    g = np.load(GOLDEN)
    inp, ref = g["inp"], g["out"]
    assert set(np.unique(inp[:, 0])) == {0, 1, 2, 3, 4}
    for name, out in (("oracle", odv.pixel_funcs(inp)), ("host build", None)):
        if out is None:
            out = np.zeros_like(ref); emu.debug_pixel_funcs_emu(np.ascontiguousarray(inp).ctypes.data, len(inp), out.ctypes.data)
        exact = inp[:, 0] != 4
        bad = np.nonzero((out != ref).any(1) & exact)[0]
        assert len(bad) == 0, f"{name}: {len(bad)} of {len(inp)} records differ, first {inp[bad[0]]} -> {out[bad[0]]} vs {ref[bad[0]]}"
        # DbgShowNormalSRGB: HLSL leaves pow's precision to the compiler and the reference build here takes glibc's powf, the library a double pow rounded once; the
        # formula around it is pinned by agreement to one ulp (observed: 5 of 3006 records differ, by one ulp)
        ulps = np.abs(out[~exact].view(np.int32).astype(np.int64) - ref[~exact].view(np.int32).astype(np.int64))
        assert ulps.max() <= 1 and (ulps == 0).all(1).mean() > 0.99, (name, int(ulps.max()))


def _unit(rng, n):
    v = rng.normal(size=(n, 3)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v


def _surfaces(n=4000, seed=3):
    rng = np.random.default_rng(seed)
    f = np.zeros((n, 28), np.float32)
    f[:, 0:2] = rng.random((n, 2))
    for k in range(5): f[:, 2 + 3 * k:5 + 3 * k] = _unit(rng, n)
    f[:8, 2:17] = np.float32([0, 0, 1, -1, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, -1])        # axis-aligned normals: pow at 0, 0.5 and 1
    f[:, 19:27] = rng.random((n, 8)).astype(np.float16).astype(np.float32)              # BSDF data: fp16 values, as the surface load rounds them
    w = f.view(np.uint32)
    w[:, 17] = rng.integers(0, 2, n); w[:, 18] = rng.integers(0, 2, n)
    w[:, 27] = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32); w[:16, 27] = np.arange(16)
    return w


@pytest.mark.parametrize("view", S.DEBUG_VIEWS_FIRST_HIT)
def test_first_hit_views_match_oracle(emu, odv, view):
    rec = _surfaces()
    out = np.zeros((len(rec), 4), np.float32)
    emu.debug_first_hit_emu(view, rec.ctypes.data, len(rec), out.ctypes.data)
    ref = odv.first_hit_records(view, rec)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), S.DEBUG_VIEW_NAMES[view]
    assert (out[:, 3] == 1).all() and np.isfinite(out).all()


def _planes(lib, W, H, seed):
    """random realtime buffers in the library's layout: a third of the branch IDs invalid, every packed word random but finite as fp16"""
    rng = np.random.default_rng(seed)
    L = lib.oracle_generic_ts_line_stride(W, H); P = lib.oracle_generic_ts_plane_stride(W, H)
    planes = np.zeros(3 * P, S.STABLE_PLANE_DTYPE)
    raw = planes.view(np.uint32).reshape(3 * P, 20)
    half = lambda shape: rng.uniform(-4, 4, shape).astype(np.float16).view(np.uint16).astype(np.uint32)
    raw[:] = half((3 * P, 20)) | (half((3 * P, 20)) << 16)
    fl = planes.view(np.float32).reshape(3 * P, 20)
    fl[:, 0:8] = rng.uniform(-50, 400, (3 * P, 8)).astype(np.float32)
    fl[::7, 7] = np.float32(1e15)                                                       # sky planes: SceneLength = kMaxRayTravel
    rad = planes["PackedNoisyRadianceAndSpecAvg"]
    rad[:] = (rng.uniform(0, 3, (3 * P, 4)).astype(np.float16).view(np.uint16).astype(np.uint32).reshape(3 * P, 2, 2) * np.uint32([1, 65536])).sum(-1)
    planes["PackedNormal"] = rng.integers(0, 2**32, 3 * P, dtype=np.uint64).astype(np.uint32)
    header = rng.integers(1, 2**20, (4, H, W), dtype=np.uint64).astype(np.uint32)
    header[:3][rng.random((3, H, W)) < 0.33] = 0xFFFFFFFF
    sr = rng.uniform(0, 5, (H, W, 4)).astype(np.float16)
    return dict(planes=planes, header=header, stable_radiance=sr, depth=np.zeros((H, W), np.float32), motion=np.zeros((H, W, 4), np.float16),
                throughput=np.zeros((H, W), np.uint32), spec_hit_t=np.zeros((H, W), np.float32)), L, P


@pytest.mark.parametrize("size", [(32, 24), (37, 19)])
def test_stable_plane_views_match_oracle(emu, odv, size):
    from rtxpt_b200 import scenes, scene_builder as sb
    W, H = size
    scene, cam = scenes.cornell_box(W, H)
    o = odv.oracle.Oracle(scene); o.set_constants(sb.make_constants(W, H, cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=8, sub_samples=1)
    buf, L, P = _planes(odv.oracle.lib(), W, H, seed=W)
    for view in S.DEBUG_VIEWS_STABLE_PLANES:
        for plane in (0, 1, 2, -1):
            out = np.zeros((H, W, 4), np.float32)
            emu.debug_stable_planes_emu(view, plane, W, H, L, P, buf["planes"].ctypes.data, buf["header"].ctypes.data, buf["stable_radiance"].ctypes.data, out.ctypes.data)
            ref = odv.stable_planes(o, rt, view, plane, buf)
            assert np.array_equal(out.view(np.uint32), ref.view(np.uint32)), (S.DEBUG_VIEW_NAMES[view], plane)
            assert (ref[..., 3] == 1).all()
    o.close()


def test_validation_mirror():
    V = S.DEBUG_VIEW
    assert S.DEBUG_VIEW_MAX_COUNT == 54 and V["FirstHit_Barycentrics"] == 29 and V["StableRadiance"] == 18 and V["ReGIRIndirectOutput"] == 53
    assert C.sizeof(S.DebugView) == 8
    for v in [V["Disabled"]] + list(S.DEBUG_VIEWS_FIRST_HIT) + list(S.DEBUG_VIEWS_STABLE_PLANES) + list(S.DEBUG_VIEWS_DENOISER_MERGE):
        for plane in (0, 1, 2, S.DEBUG_VIEW_STABLE_PLANE_SPLIT): assert S.debug_view_status(v, plane) == 0, (v, plane)
    refused = [v for v in range(S.DEBUG_VIEW_MAX_COUNT) if v not in S.DEBUG_VIEWS_FIRST_HIT + S.DEBUG_VIEWS_STABLE_PLANES + S.DEBUG_VIEWS_DENOISER_MERGE + (0,)]
    assert refused == list(range(19, 29)) + list(range(43, 54))
    for v in refused: assert S.debug_view_status(v) == -6
    for v in (54, 55, 1000, 0xFFFFFFFF): assert S.debug_view_status(v) == -1
    for plane in (3, 4, 0x7FFFFFFF, 0xFFFFFFFE): assert S.debug_view_status(V["StablePlane_Normals"], plane) == -1
