"""GPU: rtxpt_b200_update_env_map (envbake_kernels.cu + api.cu) re-bakes the environment of a live context.  The cube it leaves in the context is word for word what
rtxpt_b200_bake_env_map returns; its importance map is the host's up to libdevice's cos / sin (bars marked "measured" come from GPU runs of these tests); the light list, lookup
map, frames and NEE-AT's feedback state that follow from it are the oracle's once the oracle is given the same cube and the device's importance map.  CPU half:
tests/test_env_update.py."""
import ctypes as C
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
E = 5368


@pytest.fixture(scope="module")
def oracle(oracle):
    """The oracle module, bound for this module's tests to tests/emu's liboracle_env.so: the same oracle plus the entry points that replace a context's environment."""
    from test_env_update import env_lib, ORACLE_ENV_LIB
    env_lib(ORACLE_ENV_LIB)
    saved = oracle._lib, oracle.LIB_PATH
    oracle._lib, oracle.LIB_PATH = None, ORACLE_ENV_LIB
    oracle.lib()
    yield oracle
    oracle._lib, oracle.LIB_PATH = saved


@pytest.fixture(scope="module", params=["fast", "strict"])
def ctx(product, request):
    c = product.Context(max_sub_samples_per_launch=1, strict=(request.param == "strict"))
    c.variant = request.param
    yield c
    c.close()


def _sun(t, intensity=40.0):
    d = np.float32([np.cos(t) * 0.6, -0.55 - 0.3 * np.sin(t), np.sin(t) * 0.6]); d /= np.linalg.norm(d)
    return [((1.0, 0.92, 0.8), intensity, tuple(float(x) for x in d), 0.06)]


def _source(seed=3, h=64, w=128):
    return np.random.default_rng(seed).gamma(2.0, 0.4, (h, w, 4)).astype(np.float32)


def _flat(mips): return np.concatenate([m.ravel() for m in mips])


def _state(c):
    return [c.scene_raw(w).copy() for w in (7, 8, 9)] + [x.copy() for x in c.lights()]


def _same(a, b): return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))


def _oracle_set_env(o, cube_flat, cube_dim, chain=None):
    from oracle_lib import lib
    L = lib(); L.oracle_set_env_cube.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]; L.oracle_set_env_cube.restype = C.c_int
    cube = np.ascontiguousarray(cube_flat, np.float32); ch = None if chain is None else np.ascontiguousarray(chain, np.float32)
    assert L.oracle_set_env_cube(o.h, cube_dim, cube_dim.bit_length(), cube.ctypes.data, None if ch is None else ch.ctypes.data) == 0


def _oracle_env_maps(o, what):
    from oracle_lib import lib
    L = lib(); L.oracle_get_env_maps.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]; L.oracle_get_env_maps.restype = C.c_int64
    n = L.oracle_get_env_maps(o.h, what, None, 0); a = np.zeros(n // 4, np.float32 if what == 0 else np.uint32)
    assert L.oracle_get_env_maps(o.h, what, a.ctypes.data, a.nbytes) == n
    return a


def _host_chain(cube_mip0):
    from oracle_lib import lib
    cube = np.ascontiguousarray(cube_mip0, np.float32); out = np.zeros(sum((1024 >> m) ** 2 * 4 for m in range(11)), np.float32)
    f = lib().oracle_env_radiance_map; f.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p]; f.restype = C.c_int
    assert f(cube.shape[1], cube.ctypes.data, out.ctypes.data) == 0
    return out


def test_cube_is_the_bake(ctx, product, small_city, cornell):
    """Readback 7 after an update equals bake_env_map of the same description word for word in every MIP: across cubeDim changes, on a scene uploaded without a cube and
    when the kept source is reused.  Bad descriptions change nothing."""
    from rtxpt_b200 import scene_builder as sb
    scene, cam = small_city
    ctx.upload_scene(scene); ctx.set_constants(sb.make_constants(cam.ViewportSize[0], cam.ViewportSize[1], cam, env_enabled=True))
    src = _source()
    for i, dim in enumerate((64, 128, 64)):
        ctx.update_env_map(dim, src, scale_color=(1.0, 0.9, 1.1), lights=_sun(i))
        want = _flat(ctx.bake_env_map(dim, src, scale_color=(1.0, 0.9, 1.1), lights=_sun(i)))
        got = ctx.scene_raw(7); assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), dim
    ctx.update_env_map(64, kept_source=(1, src.shape[1], src.shape[0]), lights=_sun(5))           # the kept source, a moved sun
    assert np.array_equal(ctx.scene_raw(7).view(np.uint32), _flat(ctx.bake_env_map(64, src, lights=_sun(5))).view(np.uint32))
    # bad descriptions: the cube, the importance map, the lookup map and the light list stay
    before = _state(ctx)
    for kwargs in (dict(cube_dim=48, source=src), dict(cube_dim=64, kept_source=(1, 64, 64)), dict(cube_dim=64, kept_source=(2, 128, 128)),
                   dict(cube_dim=64, source=src, source_type=3), dict(cube_dim=8192, source=src)):
        with pytest.raises(product.RtxptError): ctx.update_env_map(**kwargs)
        assert _same(_state(ctx), before), kwargs
    # a scene uploaded without a cube gains one
    scene, cam = cornell
    ctx.upload_scene(scene); ctx.set_constants(sb.make_constants(256, 256, cam, env_enabled=True))
    assert ctx.scene_raw(7).size == 0 and ctx.scene_raw(8).size == 0
    ctx.update_env_map(32, lights=_sun(1))
    assert np.array_equal(ctx.scene_raw(7).view(np.uint32), _flat(ctx.bake_env_map(32, lights=_sun(1))).view(np.uint32))
    assert ctx.scene_raw(9).size == 1024 * 1024


@pytest.mark.parametrize("dim", [256, 1024])
def test_importance_map_against_the_host(product, oracle, small_city, dim):
    """Readback 8 against the oracle's buildEnvRadianceMap of the same cube: libdevice's cos / sin against glibc's move a tap across a texel boundary now and then."""
    from rtxpt_b200 import scene_builder as sb, lib as plib
    scene, cam = small_city
    c = product.Context(strict=True); c.upload_scene(scene); c.set_constants(sb.make_constants(cam.ViewportSize[0], cam.ViewportSize[1], cam, env_enabled=True))
    c.update_env_map(dim, _source(7, 256, 512), lights=_sun(0.4, 200.0))
    cube = plib.split_env_mips(c.scene_raw(7), dim)[0]
    got, want = plib.split_importance_mips(c.scene_raw(8)), plib.split_importance_mips(_host_chain(cube))
    for m, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, a.astype(np.float16).astype(np.float32))                          # fp16 values
        same = float((a == b).all(-1).mean()); rel = np.abs(a - b) / np.maximum(np.abs(b), 1e-3)
        close = float((rel.max(-1) <= 0.05).mean()); total = abs(float(a[..., 3].sum()) / float(b[..., 3].sum()) - 1)
        print(f"importance dim={dim} mip={m}: {100 * same:.4f} % texels bit-identical, {100 * close:.4f} % within 5 %, worst {float(rel.max()):.3g}, importance sum {total:.2e}")
        # measured (H100): MIP 0 99.64-99.71 % bit-identical, every MIP >= 93.7 % bit-identical and >= 99.96 % within 5 %, sums within 1e-6.  A tap that libdevice's cos / sin
        # move across a texel boundary at the sun changes its texel by up to 30 %; coarser MIPs average that down
        if m == 0: assert same >= 0.995, (m, same)
        assert close >= 0.98 and total < 1e-3, (m, close, total)
    c.close()


def test_light_list_and_lookup_map_follow_the_oracle(ctx, oracle, small_city, cornell):
    """Given the new cube and the device's importance map, the oracle bakes the same light list, proxy counters, proxy table and lookup map: right after the update, after
    set_constants changes the tint, rotation and importance of the environment, and after update_lights."""
    from rtxpt_b200 import scene_builder as sb
    for scene, cam in (small_city, cornell):
        W, H = cam.ViewportSize[0], cam.ViewportSize[1]
        consts = sb.make_constants(W, H, cam, env_enabled=True)
        ctx.upload_scene(scene); ctx.set_constants(consts)
        o = oracle.Oracle(scene); o.set_constants(consts)
        ctx.update_env_map(128, _source(11), lights=_sun(1.2))
        _oracle_set_env(o, ctx.scene_raw(7), 128, ctx.scene_raw(8))

        def check(stage):
            (lp, cp, pp), (lo, co, po) = ctx.lights(), o.lights()
            assert np.array_equal(lp, lo) and np.array_equal(cp, co) and np.array_equal(pp, po), stage
            assert np.array_equal(ctx.scene_raw(9), _oracle_env_maps(o, 1)), stage
            assert np.array_equal(ctx.scene_raw(8).view(np.uint32), _oracle_env_maps(o, 0).view(np.uint32)), stage
        check("update")
        consts.envMap.ColorMultiplier[:] = (0.6, 0.9, 1.4); consts.distantVsLocalImportance = 3.0
        a = 0.7; rot = [np.cos(a), 0, np.sin(a), 0, 0, 1, 0, 0, -np.sin(a), 0, np.cos(a), 0]
        consts.envMap.Transform[:] = [float(x) for x in rot]
        consts.envMap.InvTransform[:] = [float(x) for x in np.concatenate([np.array(rot, np.float32).reshape(3, 4)[:, :3].T, np.zeros((3, 1), np.float32)], 1).ravel()]
        ctx.set_constants(consts); o.set_constants(consts); check("set_constants")
        lights = sb.make_light_array([sb.point_light((1.0, 2.0, 1.5), (1.0, 0.8, 0.6), 25.0, 0.1), sb.point_light((-1.0, 1.5, 0.5), (0.6, 0.8, 1.0), 15.0, 0.2)])
        ctx.update_lights(lights); o.set_lights(lights); check("update_lights")
        o.close()


def _with_cube(scene, mips):
    """The scene's description with its environment cube replaced by `mips` (a list of 6 x n x n x 4 arrays), as an object upload_scene / Oracle take."""
    from types import SimpleNamespace
    from rtxpt_b200 import structs as S
    d = S.SceneDesc(); C.memmove(C.byref(d), C.byref(scene.desc), C.sizeof(d))
    keep = [np.ascontiguousarray(m) for m in mips]
    d.envCube.faceSize, d.envCube.mipLevels = keep[0].shape[1], len(keep)
    for m, arr in enumerate(keep):
        for f in range(6): d.envCube.faces[f][m] = arr[f].ctypes.data
    return SimpleNamespace(desc=d, keep=keep, parent=scene)


def test_frames_after_an_update_meet_the_upload_bars(ctx, oracle, small_city, cornell):
    """A reference-mode frame with the environment and a sun, rendered after an update, against the oracle given the same cube and importance map, meets the bars of a fresh
    upload of the same cube against the oracle (same ray counts in the strict build, as many bit-identical pixels, the same per-pixel L2; city: L2 <= 1e-3 at 1 spp).  The texture
    unit filters the cube with weights the oracle's software filter does not reproduce bit for bit, so a bright sun leaves fewer bit-identical pixels than a scene without one:
    measured (H100), update and upload alike, Cornell 91.1-91.3 % bit-identical with L2 1.1e-4, city 49 % with L2 2.9e-4."""
    from rtxpt_b200 import scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    for which, (scene, cam) in (("cornell", cornell), ("city", small_city)):
        W, H = cam.ViewportSize[0], cam.ViewportSize[1]
        consts = sb.make_constants(W, H, cam, bounce_count=2 if which == "cornell" else 6, diffuse_bounce_count=2 if which == "cornell" else 6, env_enabled=True,
                                   firefly_threshold=0.0 if which == "cornell" else 5000.0)
        src, sun = _source(5, 128, 256), _sun(0.9, 80.0)
        fresh = _with_cube(scene, ctx.bake_env_map(256, src, lights=sun))
        res = {}
        for kind in ("update", "upload"):
            if kind == "update":
                ctx.upload_scene(scene); ctx.set_constants(consts); ctx.update_env_map(256, src, lights=sun)
                o = oracle.Oracle(scene); o.set_constants(consts); _oracle_set_env(o, ctx.scene_raw(7), 256, ctx.scene_raw(8))
            else:
                ctx.upload_scene(fresh); ctx.set_constants(consts); o = oracle.Oracle(fresh); o.set_constants(consts)
            ctx.reset_accumulation(); ctx.path_trace(0, 1); img = ctx.readback_accumulated(); st = ctx.stats()
            acc, n, _, _, ost = o.render(0, 1); o.close()
            d = np.abs(img[..., :3] - acc[..., :3])
            res[kind] = dict(same=float((d.max(-1) == 0).mean()), l2=per_pixel_l2(img, acc), rays=(int(st.scatterRays), int(st.shadowRays)), orays=(int(ost.scatterRays), int(ost.shadowRays)))
        u, f = res["update"], res["upload"]
        print(f"frames {which} {ctx.variant}: update {u}, upload {f}")
        if ctx.variant == "strict" and which == "cornell": assert u["rays"] == u["orays"] and f["rays"] == f["orays"]
        else: assert all(abs(a - b) <= 2e-3 * b for a, b in zip(u["rays"], u["orays"]))
        assert u["same"] >= f["same"] - 0.005 and u["l2"] <= 2 * f["l2"] + 1e-7, (u, f)
        if which == "city": assert u["l2"] < 1e-3


def test_neeat_feedback_follows_the_sun(product, oracle):
    """NEE-AT with feedback while the sun moves: product and oracle go through the same frames, environment updates and update_begin / update_end calls (the oracle's reservoirs
    feed both sides, the product's depth and motion guides feed both update_ends), and the reservoirs, usage counters, proxy tables and tile lists stay bit-identical."""
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    from test_gpu_neeat import _same_state
    W, H = 90, 58
    scene, cam = scenes.light_gallery(W, H, bays=7)
    consts = sb.make_constants(W, H, cam, bounce_count=2, diffuse_bounce_count=2, env_enabled=True); consts.NEEATFeedback = 1; consts.NEEATImportanceBoost = 3
    c = product.Context(max_sub_samples_per_launch=1, strict=True, flags=S.CFG_EXPORT_GUIDES); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam)); o.neeat_reset()
    remapped = 0
    for f in range(7):
        if f % 2 == 0:                                   # the sun moves every other frame
            c.update_env_map(64, lights=_sun(0.3 * f, 120.0)); _oracle_set_env(o, c.scene_raw(7), 64, c.scene_raw(8))
        consts.sampleBaseIndex = f; c.set_constants(consts); o.set_constants(consts)
        li_p, _, px_p = c.lights(); li_o, _, px_o = o.lights(); assert np.array_equal(li_p, li_o) and np.array_equal(px_p, px_o), f
        n_lights = len(li_o)
        if f > 0:
            cand = o.neeat_raw(1, np.uint32, W * H); remapped += int(((cand != 0xFFFFFFFF) & ((cand & 0x7FFFFFFF) < E)).sum()) if f % 2 == 0 else 0
            c.neeat_set_feedback(o.neeat_raw(0, np.float32, W * H), cand)
        o.neeat_update_begin(); c.neeat_update_begin(); c.synchronize(); _same_state(c, o, W, H, n_lights, "begin")
        c.neeat_update_end(); depth, motion, _ = c.readback_guides(); o.neeat_update_end(depth, motion)
        _same_state(c, o, W, H, n_lights, "end")
        o.render(f, 1); c.path_trace(f, 1); c.synchronize()
    assert remapped > 100                                # reservoirs named environment nodes when the environment changed under them
    c.close(); o.close()
