"""GPU: realtime mode at the frame shapes, tile partitions and resizes its kernels have to handle.

The per-pixel passes of realtime mode (BUILD, FILL and the merge of realtime_kernels.cu, RTXPT's side of the denoiser interface, the DenoiseSpecHitT guide filter and
NEE-AT's feedback passes) index through 8 x 8 GenericTS tiles padded past the frame, warp-aggregated appends that run on partial warps, 16 x 16 2-D grids and
neighbour reads that clamp or mirror at the frame's edges.  The strict (IEEE) build is the oracle's bit for bit, so at every shape below the tests compare word for
word: frames smaller than a warp, pixel counts that are no multiple of 32 or 256, NEE-AT's tilesX = 3, ragged 8 x 8 and 16 x 16 tiles, and the limits set_constants
accepts.  Bars looser than bit-identical carry the value measured on an H100."""
import numpy as np
import pytest

from test_gpu_realtime import _same_headers
from test_gpu_neeat import _same_state

SHAPES = [(1, 1), (7, 5), (9, 9), (33, 17), (200, 130), (65535, 1), (1, 4097)]
BIG = (1921, 1081)
# oracle windows of the big frame (x0, y0, x1, y1): the top-left corner, the right edge (a ragged last tile column) and the bottom-right corner
BIG_WINDOWS = [(0, 0, 48, 40), (1921 - 33, 520, 1921, 560), (1921 - 41, 1081 - 33, 1921, 1081)]
STRICT = pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])


def _cuda_device_present():
    import ctypes
    try:
        cu = ctypes.CDLL("libcuda.so.1"); n = ctypes.c_int(0)
        return cu.cuInit(0) == 0 and cu.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


# GPU tests: marked for `-m gpu`, and skipped (not failed) where no device exists so that this file's CPU test runs anywhere
gpu = pytest.mark.skipif(not _cuda_device_present(), reason="needs a CUDA device")
INVALID = 0xFFFFFFFF
SENTINEL = 0xA5
FAST_SPEC_HIT_T_ULPS = 4     # two passes of up to 2 ulp each in the default build (test_spec_hit_t_filter_at_frame_shapes)
E = 5368                     # environment quad-tree nodes at the head of every light list


def _allow(pixels, share):
    """Differing pixels a bar of `share` of the frame admits, counted per frame: at least two (libdevice vs glibc sin / cos on a frame of a few pixels)."""
    return max(2, int(share * pixels))


# ---- DenoiseSpecHitT: a plain reference of specHitTNeighbourhood (guides_filter.cuh) ---------------------------------------------------------------------------
def spec_hit_t_pass(src, depth, dtype=np.float32):
    """One pass of specHitTNeighbourhood over every pixel, vectorised over pixels; per pixel the operations run in the kernel's order (x outer, y inner, centre skipped),
    each rounded to `dtype`."""
    f = dtype
    src = np.asarray(src, f); depth = np.asarray(depth, f)
    H, W = src.shape
    prev = np.maximum(f(0), src)
    prev = np.where(prev < f(5e-2), f(0), prev)
    avg = prev.copy(); sum_w = np.where(prev > 0, f(1), f(0))
    ys, xs = np.mgrid[0:H, 0:W]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for x in range(-2, 3):
            for y in range(-2, 3):
                if x == 0 and y == 0: continue
                nx, ny = xs + x, ys + y
                inside = (nx >= 0) & (ny >= 0) & (nx < W) & (ny < H)
                cx, cy = np.clip(nx, 0, W - 1), np.clip(ny, 0, H - 1)
                v = np.minimum(src[cy, cx], f(65504)); d = np.maximum(f(0), depth[cy, cx])
                ok = inside & (v > 0) & (np.abs(d - depth) <= (d + depth + f(1e-5)) * f(0.025))
                avg = np.where(ok, avg + v, avg); sum_w = np.where(ok, sum_w + f(1), sum_w)
        mean = avg / sum_w
        out = np.where(prev <= 0, mean, np.minimum(prev * f(1.5) + f(0.5), mean))
    return np.where(sum_w == 0, prev, out).astype(f)


def denoise_spec_hit_t(spec, depth, dtype=np.float32):
    """rtxpt_b200_denoise_spec_hit_t: guide -> scratch, scratch -> guide."""
    return spec_hit_t_pass(spec_hit_t_pass(spec, depth, dtype), depth, dtype)


def _bound_pairs(count=16):
    """(centre, neighbour) depths of float32 on the 2.5 % test's bound: exactly on it, one ulp inside and one ulp outside, neighbour above and below the centre."""
    f = np.float32
    exact, inside, outside = [], [], []
    for c in np.geomspace(0.3, 900.0, 4000).astype(f):
        for guess in ((f(1.025) * c + f(2.5e-7)) / f(0.975), (f(0.975) * c - f(2.5e-7)) / f(1.025)):
            d = guess + (np.arange(-64, 65) * np.spacing(guess)).astype(f)
            lhs, rhs = np.abs(d - c), (d + c + f(1e-5)) * f(0.025)
            on = np.nonzero(lhs == rhs)[0]
            if len(on) and len(exact) < count: exact.append((c, d[on[0]]))
            flip = np.nonzero((lhs[:-1] <= rhs[:-1]) != (lhs[1:] <= rhs[1:]))[0]
            for i in flip[:1]:
                a, b = (d[i], d[i + 1]) if lhs[i] <= rhs[i] else (d[i + 1], d[i])
                if len(inside) < count: inside.append((c, a)); outside.append((c, b))
        if len(exact) >= count and len(inside) >= count: break
    return np.asarray(exact, f), np.asarray(inside, f), np.asarray(outside, f)


def _spec_inputs(W, H, seed=5):
    """Synthetic depth and specular-hit-distance guides: zeros, negatives, values about the 5e-2 floor and above 65504, depth pairs on, just inside and just outside
    the 2.5 % test, and bands of rows and columns where no pixel has a valid neighbour."""
    f = np.float32
    rng = np.random.default_rng(seed + W * 7 + H)
    special = np.array([0.0, -1.0, -0.0, np.nextafter(f(5e-2), f(0)), f(5e-2), np.nextafter(f(5e-2), f(1)), 1e-3, 65504.0, 65505.0, 7e4, 1e6, 3e38], f)
    spec = rng.uniform(0.05, 60.0, (H, W)).astype(f)
    pick = rng.random((H, W)) < 0.35
    spec[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    depth = (5.0 + 0.2 * rng.standard_normal((H, W))).astype(f)
    odd = rng.random((H, W)) < 0.05
    depth[odd] = np.array([0.0, -2.0, -0.0, 1e-6], f)[rng.integers(0, 4, int(odd.sum()))]
    exact, inside, outside = _bound_pairs()
    pairs = np.concatenate([exact, inside, outside])
    k = 0
    for y in range(H):                                  # on every third row (or column of a one-pixel-wide frame) pairs of neighbours on, inside and outside the bound
        if y % 3: continue
        for x in range(0, W - 1, 2):
            depth[y, x], depth[y, x + 1] = pairs[k % len(pairs)]; k += 1
    if W == 1:
        for y in range(0, H - 1, 3):
            depth[y, 0], depth[y + 1, 0] = pairs[k % len(pairs)]; k += 1
    if H >= 12: spec[H // 2 - 2:H // 2 + 3, :] = np.where(rng.random((5, W)) < 0.5, f(0), f(-3))        # a row with no valid neighbour
    if W >= 12: spec[:, W // 2 - 2:W // 2 + 3] = np.where(rng.random((H, 5)) < 0.5, f(0), f(0.01))      # a column with none
    return depth, spec


@pytest.mark.parametrize("w,h", SHAPES + [BIG])
def test_spec_hit_t_replay_is_the_oracle(oracle, w, h):
    """CPU: the float32 replay equals the oracle's DenoiseSpecHitT bit for bit at every shape; the float64 reference agrees where no value sits on a decision."""
    depth, spec = _spec_inputs(w, h)
    got = denoise_spec_hit_t(spec, depth)
    want = oracle.denoise_spec_hit_t(depth, spec)
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32)), (w, h, int((got.view(np.uint32) != want.view(np.uint32)).sum()))
    # float64 sanity bar on guides without planted decisions (smooth depth, hit distances well inside their ranges)
    rng = np.random.default_rng(w + 3 * h)
    d2 = rng.uniform(4.0, 6.0, (h, w)).astype(np.float32); s2 = rng.uniform(0.1, 100.0, (h, w)).astype(np.float32)
    a, b = denoise_spec_hit_t(s2, d2), denoise_spec_hit_t(s2, d2, np.float64)
    assert np.allclose(a, b, rtol=1e-5, atol=0), float(np.abs(a / b - 1).max())
    assert (got[spec > 0] >= 0).all()


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def _upload(c, buffer, array):
    from reblur_inputs import upload
    upload(c, buffer, array)


def _cornell(W, H):
    from rtxpt_b200 import scenes
    return scenes.cornell_box(W, H, delta_surfaces=True)


def _context(product, strict, W, H, scene=None, cam=None, sub_samples=1, bounces=8, **kw):
    from rtxpt_b200 import scene_builder as sb
    if scene is None: scene, cam = _cornell(W, H)
    consts = sb.make_constants(W, H, cam, bounce_count=bounces, diffuse_bounce_count=3)
    c = product.Context(max_sub_samples_per_launch=1, strict=strict, **kw); c.upload_scene(scene); c.set_constants(consts); c.set_view(sb.world_to_clip(cam))
    rt = sb.make_realtime_constants(W, H, cam, bounce_count=bounces, sub_samples=sub_samples); c.set_realtime(rt)
    return c, consts, rt


@pytest.mark.gpu
@gpu
@STRICT
@pytest.mark.parametrize("w,h", SHAPES)
def test_spec_hit_t_filter_at_frame_shapes(product, w, h, strict):
    """k_dn_spec_hitt on synthetic guides written through the context's buffers: the strict build is the float32 replay bit for bit.  The default build (FMA in
    prevHitT * 1.5 + 0.5, approximate division) is within 2 ulp of the replay in one pass; the second pass averages first-pass values that are each up to 2 ulp off
    and adds its own 2, so the two passes are held to 4 ulp.  measured (H100 SXM, 700 W): strict 0 ulp at every shape; default build at most 2 ulp up to 9 x 9
    and on 1 x 4097, 3 ulp at 33 x 17, 4 ulp at 200 x 130 and 65535 x 1 (14 % of the pixels of 65535 x 1 differ)."""
    from rtxpt_b200 import structs as S
    c, _, _ = _context(product, strict, w, h)
    try:
        depth, spec = _spec_inputs(w, h)
        _upload(c, S.BUFFER_DEPTH_F32, depth); _upload(c, S.BUFFER_SPECULAR_HITT_F32, spec)
        c.denoise_spec_hit_t(); c.synchronize()
        got = c.readback_realtime()["spec_hit_t"]
        want = denoise_spec_hit_t(spec, depth)
        worst = int(_ulps(got, want).max())
        print("spec hit t %dx%d %s: %d pixels differ from the float32 replay, at most %d ulp" % (w, h, "strict" if strict else "fast", int((got != want).sum()), worst))
        if strict: assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (w, h, int((got != want).sum()))
        else: assert worst <= FAST_SPEC_HIT_T_ULPS, (w, h, worst)
    finally:
        c.close()


# ---- BUILD + FILL + merge ----------------------------------------------------------------------------------------------------------------------------------------
def _padding_mask(W, H):
    """Plane-buffer entries that no in-frame pixel maps to (GenericTS padding of the ragged last tile column and row)."""
    from rtxpt_b200 import scene_builder as sb
    stride = ((W + 7) // 8) * 8 * ((H + 7) // 8) * 8
    pad = np.ones(3 * stride, bool)
    ys, xs = np.mgrid[0:H, 0:W]
    for plane in range(3):
        pad[sb.generic_ts_address(xs.ravel(), ys.ravel(), plane, W, H)] = False
    return pad


def _fill_sentinel(c):
    from rtxpt_b200 import structs as S
    _, nbytes = c.device_ptr(S.BUFFER_STABLE_PLANES)
    _upload(c, S.BUFFER_STABLE_PLANES, np.full(nbytes, SENTINEL, np.uint8))


def _check_sentinel(g, W, H, pad):
    """The padding still holds the sentinel; every valid in-frame record was written in full (each of its five 16-byte words differs from the sentinel)."""
    from rtxpt_b200 import scene_builder as sb
    raw = g["planes"].view(np.uint8).reshape(-1, 80)
    assert (raw[pad] == SENTINEL).all(), ("padding written", int((raw[pad] != SENTINEL).any(1).sum()))
    ys, xs = np.mgrid[0:H, 0:W]
    for plane in range(3):
        v = g["header"][plane] != INVALID
        rec = raw[sb.generic_ts_address(xs[v], ys[v], plane, W, H)].reshape(-1, 5, 16)
        assert not (rec == SENTINEL).all(-1).any(), ("valid record left unwritten", plane, int((rec == SENTINEL).all(-1).any(-1).sum()))


def _compare_frame(g, r, W, H, strict, sub_samples, mask):
    """The bars of test_realtime_strict_build_is_the_oracle, test_build_pass_matches_oracle and test_fill_pass_and_merge_match_oracle, counted per frame on `mask`."""
    from rtxpt_b200 import scene_builder as sb
    P = int(mask.sum())
    same = _same_headers(g, r, strict) & mask
    ys, xs = np.nonzero(same)
    if strict:
        differ = (g["header"] != r["header"]).any(0) & mask
        for k in ("stable_radiance", "depth", "motion", "throughput", "spec_hit_t"):
            a, b = g[k], r[k]
            differ |= (a.view(np.uint8).reshape(H, W, -1) != b.view(np.uint8).reshape(H, W, -1)).any(-1) & mask
        noisy = 0
        for plane in range(3):
            v = r["header"][plane][ys, xs] != INVALID
            addr = sb.generic_ts_address(xs[v], ys[v], plane, W, H)
            a, b = g["planes"][addr], r["planes"][addr]
            if not len(a): continue
            bad = np.zeros(len(a), bool)
            for f in a.dtype.names:
                if f == "PackedNoisyRadianceAndSpecAvg": noisy += int((a[f] != b[f]).any(-1).sum()); continue
                x, y = a[f].reshape(len(a), -1), b[f].reshape(len(b), -1)
                if x.dtype.kind == "u": bad |= (x != y).any(1)
                else: bad |= ~np.isclose(x, y, rtol=1e-6, atol=1e-6, equal_nan=True).all(1)
            differ[ys[v][bad], xs[v][bad]] = True
        print("  strict: %d of %d pixels differ in header / plane record / guides, %d noisy-radiance words" % (int(differ.sum()), P, noisy))
        assert differ.sum() <= _allow(P, 0.005), (W, H, int(differ.sum()))
        assert noisy <= _allow(P, 0.005 if sub_samples == 1 else 0.04), (W, H, noisy)
        d = np.abs(g["merged"] - r["merged"])[same]; scale = np.maximum(r["merged"][same], 0.05)
        assert (d != 0).any(-1).sum() <= _allow(P, 0.005 if sub_samples == 1 else 0.03), (W, H, int((d != 0).any(-1).sum()))
        assert (d / scale >= 0.05).any(-1).sum() <= _allow(P, 0.005), (W, H)
        return
    assert (mask & ~same).sum() <= _allow(P, 0.02), (W, H, int((mask & ~same).sum()))
    for plane in range(3):
        v = r["header"][plane][ys, xs] != INVALID
        addr = sb.generic_ts_address(xs[v], ys[v], plane, W, H)
        a, b = g["planes"][addr], r["planes"][addr]
        if not len(a): continue
        assert (a["VertexIndexAndRoughness"] >> 16 == b["VertexIndexAndRoughness"] >> 16).all(), plane
        fin = np.isfinite(b["SceneLength"]); assert (np.isfinite(a["SceneLength"]) == fin).all(), plane
        for f in ("RayOrigin", "RayDir", "SceneLength", "LastRayTCurrent"):
            if not fin.any(): break
            close = np.isclose(a[f][fin], b[f][fin], rtol=2e-4, atol=2e-3).reshape(int(fin.sum()), -1).all(1)
            assert (~close).sum() <= _allow(P, 0.005), (plane, f, int((~close).sum()))
        na, nb = a["PackedNormal"].astype(np.int64), b["PackedNormal"].astype(np.int64)
        far = (np.abs((na & 0xFFFF) - (nb & 0xFFFF)) > 8) | (np.abs((na >> 16) - (nb >> 16)) > 8)
        assert far.sum() <= _allow(P, 0.001), (plane, int(far.sum()))
    sa, sb_ = g["stable_radiance"][same].astype(np.float32), r["stable_radiance"][same].astype(np.float32)
    assert np.allclose(sa, sb_, rtol=2e-3, atol=1e-3)
    assert np.allclose(g["depth"][same], r["depth"][same], rtol=1e-5, atol=1e-6)
    assert (g["throughput"][same] != r["throughput"][same]).sum() <= _allow(P, 0.01)
    assert np.allclose(g["motion"][same].astype(np.float32), r["motion"][same].astype(np.float32), atol=2e-3)
    assert (~np.isclose(g["spec_hit_t"][same], r["spec_hit_t"][same], rtol=1e-3, atol=1e-3)).sum() <= _allow(P, 0.01)
    if sub_samples > 1:
        d = np.abs(g["merged"] - r["merged"])[same]; scale = np.maximum(r["merged"][same], 0.05)
        assert (d / scale >= 0.02).any(-1).sum() <= _allow(P, 0.1), (W, H, int((d / scale >= 0.02).any(-1).sum()))


@pytest.mark.gpu
@gpu
@STRICT
@pytest.mark.parametrize("w,h", SHAPES + [BIG])
def test_build_fill_and_merge_match_oracle_at_frame_shapes(product, oracle, w, h, strict):
    """BUILD with 1 and then 3 FILL sub-samples and the no-denoiser merge against the oracle (the big ragged frame in three windows the oracle renders), with the
    plane buffer's padding holding a sentinel the frame must not touch; then DenoiseSpecHitT on the frame's own guide against the float32 replay.  measured (H100 SXM,
    700 W): in the strict build no pixel of any shape or window differs in a header word, a plane record or a guide; the noisy radiance the FILL pass deposits
    differs in at most 21 plane words (200 x 130, 3 sub-samples: libdevice vs glibc in the BSDF sampling)."""
    from rtxpt_b200 import scene_builder as sb
    scene, cam = _cornell(w, h)
    c, consts, _ = _context(product, strict, w, h, scene, cam)
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    pad = _padding_mask(w, h)
    windows = BIG_WINDOWS if (w, h) == BIG else [(0, 0, w, h)]
    try:
        for sub in (1, 3):
            rt = sb.make_realtime_constants(w, h, cam, bounce_count=8, sub_samples=sub)
            c.set_realtime(rt); _fill_sentinel(c)
            c.path_trace_realtime(True); c.synchronize(); g = c.readback_realtime()
            _check_sentinel(g, w, h, pad)
            for win in windows:
                x0, y0, x1, y1 = win
                mask = np.zeros((h, w), bool); mask[y0:y1, x0:x1] = True
                print("%dx%d %s, %d sub-samples, window %s" % (w, h, "strict" if strict else "fast", sub, win))
                r = o.render_realtime(rt, rect=None if (w, h) != BIG else win)
                _compare_frame(g, r, w, h, strict, sub, mask)
        want = denoise_spec_hit_t(g["spec_hit_t"], g["depth"])
        c.denoise_spec_hit_t(); c.synchronize(); got = c.readback_realtime()["spec_hit_t"]
        if strict: assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got != want).sum())
        else: assert int(_ulps(got, want).max()) <= FAST_SPEC_HIT_T_ULPS, int(_ulps(got, want).max())
    finally:
        c.close(); o.close()


# ---- denoiser interface --------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@gpu
@STRICT
@pytest.mark.parametrize("w,h", SHAPES)
def test_denoiser_interface_matches_oracle_at_frame_shapes(product, oracle, w, h, strict):
    """Per plane 2, 1, 0: prepare the NRD inputs and merge with the identity denoiser, as test_denoiser_interface_matches_oracle does at 96 x 96.  The edge pixels of
    every frame read clamped neighbours in ComputeDisocclusionRelaxation; at W = 1 or H = 1 every neighbour across the thin side is the pixel itself.  The camera looks
    into the glass box from close by, so that the frame's edges lie on planes past the first vertex, the only ones whose relaxation reads neighbours."""
    from rtxpt_b200 import scene_builder as sb
    scene = _cornell(w, h)[0]
    cam = sb.bridge_camera(w, h, pos=(1.85, 0.8, -1.0), direction=(0, 0, 1), up=(0, 1, 0), fov_y=0.3)
    c, consts, _ = _context(product, strict, w, h, scene, cam)
    o = oracle.Oracle(scene); o.set_constants(consts); o.set_view(sb.world_to_clip(cam))
    try:
        rt = sb.make_realtime_constants(w, h, cam, bounce_count=8, sub_samples=2)
        c.set_realtime(rt); c.path_trace_realtime(False); c.synchronize()
        g = c.readback_realtime(); r = o.render_realtime(rt)
        k = sb.make_denoiser_constants(cam, suppress_primary_indirect_specular_k=0.4)
        d = o.new_denoiser_targets()
        P = w * h
        same = _same_headers(g, r, strict)
        # a pixel's disocclusion relaxation reads its four clamped neighbours: compare it where they decompose alike too
        sp = np.pad(same, 1, mode="edge")
        same_nb = same & sp[:-2, 1:-1] & sp[2:, 1:-1] & sp[1:-1, :-2] & sp[1:-1, 2:]
        for i, plane in enumerate((2, 1, 0)):
            c.denoiser_prepare_inputs(plane, i == 0, k); c.synchronize(); gi = c.readback_denoiser_inputs()
            o.denoiser_prepare_inputs(rt, k, r, d, plane, i == 0)
            assert np.array_equal(gi["view_z"][same] < 1e30, d["view_z"][same] < 1e30), plane
            surf = same & (d["view_z"] < 1e30)
            if strict:
                for key in ("view_z", "normal_roughness", "motion"):
                    a, b = gi[key][surf], d[key][surf]
                    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (plane, key, int((a != b).reshape(len(a), -1).any(1).sum()))
                dm = np.abs(gi["disocclusion_mix"].astype(int) - d["disocclusion_mix"])
                assert (dm[same_nb & surf] <= 1).all(), (plane, int((dm[same_nb & surf] > 1).sum()))
            else:
                assert np.allclose(gi["view_z"][surf], d["view_z"][surf], rtol=1e-5), plane
                assert (gi["normal_roughness"][surf] != d["normal_roughness"][surf]).sum() <= _allow(P, 0.01), plane
                assert np.allclose(gi["motion"][surf].astype(np.float32), d["motion"][surf].astype(np.float32), atol=1e-3), plane
                dm = np.abs(gi["disocclusion_mix"][surf].astype(int) - d["disocclusion_mix"][surf]) <= 1
                assert (~dm).sum() <= _allow(P, 0.1), (plane, int((~dm).sum()))
            for key in ("diff", "spec"):
                a, b = gi[key][surf].astype(np.float32), d[key][surf].astype(np.float32)
                far = ~np.isclose(a, b, rtol=2e-2, atol=2e-3).all(-1)
                assert far.sum() <= _allow(P, 0.03 if strict else 0.1), (plane, key, int(far.sum()))
            c.denoiser_final_merge(plane); o.denoiser_final_merge(rt, r, d, plane, d["diff"].copy(), d["spec"].copy())
        c.synchronize()
        out = c.readback_output_color().astype(np.float32); ref = d["output"].astype(np.float32)
        far = ~np.isclose(out[same], ref[same], rtol=2e-2, atol=4e-3).all(-1)
        assert far.sum() <= _allow(P, 0.03 if strict else 0.1), int(far.sum())
    finally:
        c.close(); o.close()


# ---- NEE-AT's passes ----------------------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def env_oracle(oracle):
    """The oracle bound to its build with the entry points that replace a context's environment (as in test_gpu_env_update)."""
    from test_env_update import env_lib, ORACLE_ENV_LIB
    env_lib(ORACLE_ENV_LIB)
    saved = oracle._lib, oracle.LIB_PATH
    oracle._lib, oracle.LIB_PATH = None, ORACLE_ENV_LIB
    oracle.lib()
    yield oracle
    oracle._lib, oracle.LIB_PATH = saved


@pytest.mark.gpu
@gpu
@pytest.mark.parametrize("w,h", SHAPES)
def test_neeat_passes_match_oracle_at_frame_shapes(product, env_oracle, w, h):
    """The reference-mode protocol of test_neeat_feedback_follows_the_sun (the oracle's reservoirs feed both sides, the product's depth and motion guides feed both
    update_ends) at the frame shapes: four frames with the environment off (its 5368 quad-tree nodes weigh nothing), four with it on, then three frames of synthetic
    feedback given to both sides - every pixel naming one light, every pixel invalid, and SSC candidates at the 1e12 weight cap.  Reservoirs, proxy counters, proxy
    table, blended images and tile lists stay bit-identical after every update_begin and update_end."""
    from rtxpt_b200 import scene_builder as sb, scenes, structs as S
    from test_gpu_env_update import _sun, _oracle_set_env
    oracle = env_oracle
    scene, cam = scenes.light_gallery(w, h, bays=7)
    consts = {on: sb.make_constants(w, h, cam, bounce_count=2, diffuse_bounce_count=2, env_enabled=on) for on in (False, True)}
    for k in consts.values(): k.NEEATFeedback = 1; k.NEEATImportanceBoost = 3
    c = product.Context(max_sub_samples_per_launch=1, strict=True, flags=S.CFG_EXPORT_GUIDES); c.upload_scene(scene); c.set_constants(consts[False]); c.set_view(sb.world_to_clip(cam))
    o = oracle.Oracle(scene); o.set_constants(consts[False]); o.set_view(sb.world_to_clip(cam)); o.neeat_reset()
    P = w * h
    rng = np.random.default_rng(w * 31 + h)
    try:
        for f in range(11):
            env = f >= 4
            if f == 4:
                c.update_env_map(64, lights=_sun(0.7, 120.0)); _oracle_set_env(o, c.scene_raw(7), 64, c.scene_raw(8))
            k = consts[env]; k.sampleBaseIndex = f; c.set_constants(k); o.set_constants(k)
            li_p, _, px_p = c.lights(); li_o, _, px_o = o.lights(); assert np.array_equal(li_p, li_o) and np.array_equal(px_p, px_o), f
            n_lights = len(li_o); assert n_lights > E
            if f >= 8:                                       # synthetic feedback, given to both sides
                first = E                                    # the gallery's first emissive triangle
                if f == 8: wgt, cand = np.ones(P, np.float32), np.full(P, first, np.uint32)
                elif f == 9: wgt, cand = np.zeros(P, np.float32), np.full(P, INVALID, np.uint32)
                else: wgt, cand = np.full(P, 1e12, np.float32), (rng.integers(0, n_lights, P).astype(np.uint32) | np.uint32(0x80000000))
                c.neeat_set_feedback(wgt, cand); o.neeat_set_feedback(wgt, cand)
            elif f > 0:
                c.neeat_set_feedback(o.neeat_raw(0, np.float32, P), o.neeat_raw(1, np.uint32, P))
            o.neeat_update_begin(); c.neeat_update_begin(); c.synchronize(); _same_state(c, o, w, h, n_lights, "begin")
            c.neeat_update_end(); depth, motion, _ = c.readback_guides(); o.neeat_update_end(depth, motion)
            _same_state(c, o, w, h, n_lights, "end")                 # "end" adds the processed and blended reservoirs and the tile lists
            o.render(f, 1); c.path_trace(f, 1); c.synchronize()
    finally:
        c.close(); o.close()


# ---- tile partitions -------------------------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@gpu
@STRICT
@pytest.mark.parametrize("w,h,world,tile", [(200, 130, 3, 64), (64, 64, 4, 64), (33, 17, 2, 16)])
def test_realtime_tile_partitions_at_ragged_shapes(product, w, h, world, tile, strict):
    """realtime_mgpu.realtime_frame over ranks of unequal size (200 x 130 over three), ranks that own no pixel (64 x 64 over four) and ragged 16-pixel tiles (33 x 17 over
    two): two frames bit-identical to one context's in the denoiser inputs, the ReBLUR outputs, the output colour and the LDR image; every call of an empty rank succeeds."""
    from rtxpt_b200 import scene_builder as sb, structs as S, realtime_mgpu as M
    scene, cam = _cornell(w, h)
    k = sb.make_denoiser_constants(cam); tm = S.make_tone_mapping_params(op=5, auto_exposure=True)
    one = _context(product, strict, w, h, scene, cam, sub_samples=2, bounces=6)[0]
    ranks = [_context(product, strict, w, h, scene, cam, sub_samples=2, bounces=6, tile_rank=r, tile_world=world, tile_size=tile)[0] for r in range(world)]
    try:
        owned = [p.tile_layout()[0] for p in ranks]
        assert sum(owned) == w * h
        if w * h <= tile * tile: assert owned[1:] == [0] * (world - 1)
        group = M.LocalGroup(ranks)
        for f in range(2):
            frame = sb.make_reblur_frame(cam, cam, frame_index=f)
            one.path_trace_realtime(False); one.denoise_realtime(k, frame); one.tone_map(tm); one.synchronize()
            M.realtime_frame(group, k, frame, tm)
            for p in ranks: p.synchronize()
            ref = dict(inputs=one.readback_denoiser_inputs(), reblur=one.readback_reblur(), color=one.readback_output_color(), ldr=one.readback_ldr())
            for r, p in enumerate(ranks):
                for key in ("inputs", "reblur"):
                    got = p.readback_denoiser_inputs() if key == "inputs" else p.readback_reblur()
                    for name in ref[key]: assert ref[key][name].tobytes() == got[name].tobytes(), (f, r, key, name)
                assert ref["color"].tobytes() == p.readback_output_color().tobytes() and ref["ldr"].tobytes() == p.readback_ldr().tobytes(), (f, r)
    finally:
        for p in [one] + ranks: p.close()


# ---- resizing a live context ---------------------------------------------------------------------------------------------------------------------------------------
def _frames(c, scene, cam, W, H, base):
    """Two realtime frames with ReBLUR and tone mapping, then two with NEE-AT feedback; everything each frame leaves behind."""
    from rtxpt_b200 import scene_builder as sb, structs as S
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=3)
    k = sb.make_denoiser_constants(cam); tm = S.make_tone_mapping_params(op=5, auto_exposure=True)
    c.set_constants(consts); c.set_view(sb.world_to_clip(cam)); c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2))
    out = []
    for f in range(4):
        consts.sampleBaseIndex = base + 2 * f; consts.NEEATFeedback = 1 if f >= 2 else 0; c.set_constants(consts)
        if f >= 2: c.neeat_update_begin()
        c.path_trace_realtime(False); c.denoise_realtime(k, sb.make_reblur_frame(cam, cam, frame_index=base + f)); c.tone_map(tm); c.synchronize()
        g = c.readback_realtime()
        out.append(dict(realtime={n: g[n] for n in ("header", "planes", "stable_radiance", "depth", "motion", "throughput", "spec_hit_t")}, inputs=c.readback_denoiser_inputs(),
                        reblur=c.readback_reblur(), color=c.readback_output_color(), ldr=c.readback_ldr()))
    return out


@pytest.mark.gpu
@gpu
@STRICT
def test_resizing_a_live_context_equals_a_fresh_one(product, strict):
    """One context through 96 x 96 -> 7 x 5 -> 200 x 130 -> 96 x 96, realtime frames with ReBLUR, tone mapping and then NEE-AT feedback at each size: every frame bit-identical
    to a fresh context created at that size and given the same calls (the resets of set_realtime, denoiser_prepare_inputs, neeatEnsure and ReBLUR's history)."""
    scene = _cornell(96, 96)[0]
    live = product.Context(max_sub_samples_per_launch=1, strict=strict); live.upload_scene(scene)
    try:
        for step, (W, H) in enumerate(((96, 96), (7, 5), (200, 130), (96, 96))):
            cam = _cornell(W, H)[1]
            got = _frames(live, scene, cam, W, H, 10 * step)
            fresh = product.Context(max_sub_samples_per_launch=1, strict=strict); fresh.upload_scene(scene)
            try:
                want = _frames(fresh, scene, cam, W, H, 10 * step)
            finally:
                fresh.close()
            for f, (a, b) in enumerate(zip(got, want)):
                for key in b:
                    if isinstance(b[key], dict):
                        for name in b[key]: assert a[key][name].tobytes() == b[key][name].tobytes(), (W, H, f, key, name)
                    else: assert a[key].tobytes() == b[key].tobytes(), (W, H, f, key)
    finally:
        live.close()
