"""Approximate light-vs-BSDF MIS (RtxptPathTracerConstants::useApproximateMIS = 1, RTXPT's RTXPT_USE_APPROXIMATE_MIS) held to the reference's shader code on the CPU.

tests/golden/hit_golden_amis.npz holds path vertices of the three passes (reference, BUILD, FILL) run through the UNMODIFIED PathTracer.hlsli / PathTracerNEE.hlsli / LightSampler.hlsli
compiled with the macro at 1 (tests/golden/make_hit_golden_amis.py).  The approximate-MIS oracle (oracle/amis.mk, tests/oracle_amis_lib.py) and the host build of shade.cuh's AMIS
instantiations (tests/emu/approximate_mis_host_emu.cu) must reproduce them bit for bit; a render with approximate MIS must converge to the full-MIS image; and an emitter that NEE cannot pick is weighted on the BSDF side anyway, as in RTXPT."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest
from test_shade_port import PAYLOAD, SHADOW, FEEDBACK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hit_golden_amis.npz")
COLS = {0: [c for c in PAYLOAD if c != 15] + SHADOW + FEEDBACK, 2: PAYLOAD + SHADOW + [37] + FEEDBACK + list(range(41, 51)),
        1: PAYLOAD + [29, 31] + list(range(47, 51)) + list(range(52, 56)) + list(range(56, 116))}


@pytest.fixture(scope="module")
def oracle():
    """the approximate-MIS oracle; with useApproximateMIS = 0 it is the full-MIS oracle"""
    import oracle_amis_lib
    oracle_amis_lib.build()
    return oracle_amis_lib.oracle


def _oracle_hit(oracle, u, mode):
    O = oracle.lib(); O.oracle_hit_funcs.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]; O.oracle_hit_funcs.restype = None
    u = np.ascontiguousarray(u, np.float32); out = np.zeros((len(u), 128), np.float32)
    O.oracle_hit_funcs(u.ctypes.data, len(u), out.ctypes.data, mode)
    return out


def _emu(fn_name, mk, u, mode):
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s"] + (["-f", mk] if mk else ["_build/libshade_emu.so"]), check=True)
    L = C.CDLL(os.path.join(ROOT, "tests", "emu", "_build", "libapproximate_mis_emu.so" if mk else "libshade_emu.so"))
    fn = getattr(L, fn_name); fn.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]; fn.restype = None
    u = np.ascontiguousarray(u, np.float32); out = np.zeros((len(u), 128), np.float32); st = np.zeros(len(u), np.int32)
    fn(u.ctypes.data, len(u), out.ctypes.data, st.ctypes.data, mode)
    return out, st == 0


def test_oracle_matches_approximate_mis_golden(oracle):
    """All three passes, every record (hits, misses, EmptyPathInitialize; NEE-AT feedback; NEEFullSamples 1 .. 63): the oracle with useApproximateMIS = 1 equals the reference compiled
    with RTXPT_USE_APPROXIMATE_MIS = 1 on every word; the same records with full MIS come out different, so the golden pins the approximate weights."""
    g = np.load(GOLDEN)
    for key, mode in (("hit", 0), ("build", 1), ("fill", 2)):
        u, ref = g[key + "_in"], g[key + "_out"]
        assert (u[:, 94] == 1).all()
        out = _oracle_hit(oracle, u, mode)
        same = out.view(np.uint32) == ref.view(np.uint32); same[:, 35:37] = True            # 35, 36: call counts of the stub's ExportSpecHitT hooks (not mirrored)
        if mode == 1: same[:, 30] = True; same[:, 32:35] = True; same[:, 117:120] = True    # what the stub's Export hooks were handed (as test_oracle_golden)
        assert same.all(), (key, np.argwhere(~same)[:8])
        full = u.copy(); full[:, 94] = 0
        differs = (_oracle_hit(oracle, full, mode).view(np.uint32)[:, :20] != ref.view(np.uint32)[:, :20]).any(1)
        if mode == 1: assert not differs.any()                                              # the BUILD pass evaluates no MIS
        else: assert differs.mean() > 0.25, (key, differs.mean())
        if mode != 1: assert (u[:, 84] > 8).sum() > 10 and ((u[:, 84] > 1) & (u[:, 92] == 0) & (u[:, 27] == 0)).sum() > 20 and (u[:, 92] != 0).mean() > 0.4


def test_approximate_mis_oracle_is_the_full_mis_oracle_with_the_switch_off(oracle):
    """liboracle_amis.so at useApproximateMIS = 0 reproduces the full-MIS golden hit_golden.npz (the three passes, every word test_oracle_golden compares) bit for bit, as
    liboracle.so does: the switch only adds branches."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "hit_golden.npz"))
    for key, mode in (("hit", 0), ("build", 1), ("fill", 2)):
        u, ref = g[key + "_in"], g[key + "_out"]
        assert (u[:, 94] == 0).all()
        same = _oracle_hit(oracle, u, mode).view(np.uint32) == ref.view(np.uint32); same[:, 35:37] = True
        if mode == 1: same[:, 30] = True; same[:, 32:35] = True; same[:, 117:120] = True
        assert same.all(), (key, np.argwhere(~same)[:8])


def test_shade_source_matches_approximate_mis_golden():
    """The host build of shade.cuh: shadeHit / shadeMiss< .., AMIS > in reference mode (NEE-AT instantiation) and the FILL pass, one shadow record per vertex for NEEFullSamples <= 1
    (with feedback insertion) and the multi-sample shade + NEE block for 2 .. 63 (without feedback, which the product refuses with several samples); the BUILD pass, which
    evaluates no MIS, through its one kernel body (tests/emu/shade_host_emu.cu) - bit for bit against the golden."""
    g = np.load(GOLDEN)
    for key, mode in (("hit", 0), ("fill", 2)):
        u, ref = g[key + "_in"], g[key + "_out"]
        out, ran = _emu("amis_emu_vertices", "approximate_mis.mk", u, mode)
        vertex = u[:, 27] <= 1
        assert (ran == (vertex & ~((u[:, 84] > 1) & (u[:, 92] != 0)))).all()
        same = ref.view(np.uint32)[:, COLS[mode]] == out.view(np.uint32)[:, COLS[mode]]
        assert same[ran].all(), (key, np.argwhere(~same[ran])[:8])
        multi = ran & (u[:, 84] > 1) & (u[:, 27] == 0)
        assert ran.sum() > 80 and multi.sum() > 20 and (ref[multi, 20] > 1).any(), (key, ran.sum(), multi.sum())
    u, ref = g["build_in"], g["build_out"]
    out, ran = _emu("shade_emu_vertices", None, u, 1)
    same = ref.view(np.uint32)[:, COLS[1]] == out.view(np.uint32)[:, COLS[1]]
    assert ran.sum() > 50 and same[ran].all(), np.argwhere(~same[ran])[:8]


def test_emitter_without_light_record_is_weighted_on_the_bsdf_side(oracle):
    """An emissive surface NEE cannot pick (ExcludeFromNEE, light-list overflow: no light record, neeTriangleLightIndex invalid) reached by a BSDF ray after a vertex that sampled lights:
    full MIS gives it weight 1 (shade.cuh tests the index); approximate MIS tests no index (PathTracer.hlsli:619-620) and weights it with
    bsdfPdf / (bsdfPdf + 3 x fullSamples x candidates) like any other emitter - the reference's behaviour, reproduced rather than corrected.  Pinned on the golden's records of that kind."""
    g = np.load(GOLDEN)
    for key, mode in (("hit", 0), ("fill", 2)):
        u, ref = g[key + "_in"], g[key + "_out"]
        U = u.view(np.uint32); mis = U[:, 18] >> 16; pdf = (U[:, 17] & 0xFFFF).astype(np.uint16).view(np.float16)
        sel = (u[:, 27] == 0) & (u[:, 54:57] > 0).any(1) & (u[:, 75] < 0) & ((mis & (1 << 15)) != 0) & (pdf != 0) & (u[:, 94] == 1)
        if mode == 2: sel &= ((U[:, 19] >> 10) & (1 << 17)) == 0          # FILL: a path on a stable branch adds no emission (the BUILD pass captured it)
        assert sel.sum() >= 5, (key, sel.sum())
        amis = _oracle_hit(oracle, u[sel], mode); full_u = u[sel].copy(); full_u[:, 94] = 0; full = _oracle_hit(oracle, full_u, mode)
        assert (amis.view(np.uint32)[:, :20] == ref[sel].view(np.uint32)[:, :20]).all()
        # the emitted radiance enters L (reference mode) or the noisy radiance (FILL) with weight w < 1 under approximate MIS, 1 under full MIS: the outgoing L words differ
        La, Lf = amis.view(np.uint32)[:, 10:12], full.view(np.uint32)[:, 10:12]
        assert (La != Lf).any(1).mean() > 0.5, (key, (La != Lf).any(1).mean())
        w = pdf[sel].astype(np.float32) / (pdf[sel].astype(np.float32) + np.float32(3) * (mis[sel] & 0x3F) * ((mis[sel] >> 6) & 0x3F))
        assert (w < 1).all() and (w > 0).all()


def test_approximate_mis_render_converges_to_full_mis(oracle):
    """Cornell box with its emissive quad, a sphere light with its proxy geometry, a spot light and the sky environment behind the open side: with approximate MIS the two weights of
    a direction still sum to one, so the 256-spp image agrees with the full-MIS one within sampling noise (measured by two full-MIS images of different sample indices), and is
    not the same image."""
    from rtxpt_b200 import scene_builder as sb, scenes
    b = scenes.cornell_builder(analytic_lights=True); b.set_env_cube(scenes.sky_cube(32, sun_intensity=4.0)); scene = b.build()
    W = H = 48
    cam = sb.bridge_camera(W, H, pos=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.66)
    o = oracle.Oracle(scene)

    def render(approx, base, spp=256):
        o.set_constants(sb.make_constants(W, H, cam, bounce_count=3, diffuse_bounce_count=3, env_enabled=True, sample_base_index=base, approximate_mis=approx))
        return o.render(0, spp)[0][..., :3].astype(np.float64)

    full_a, full_b, amis = render(False, 0), render(False, 100000), render(True, 200000)
    differs = not np.array_equal(render(True, 0, 16), render(False, 0, 16))
    o.close()
    blocks = lambda img: img.reshape(H // 8, 8, W // 8, 8, 3).mean((1, 3))
    noise = np.sqrt(((blocks(full_a) - blocks(full_b)) ** 2).mean())
    err = np.sqrt(((blocks(full_a) - blocks(amis)) ** 2).mean())
    assert err < 2.5 * noise, (err, noise)
    assert abs(amis.mean() / full_a.mean() - 1) < 0.02, (amis.mean(), full_a.mean())
    assert differs
