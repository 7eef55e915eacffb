"""GPU: the wavefront at every launch configuration and frame shape it accepts.

The three traversal kernels run one persistent loop (kernels.cu: traceLoop) and are launched from one table (kTraceKernels), one instantiation per
trace kind and resident-CTA count; RTXPT_TRACE_CTAS picks the column, and kinds without a MINB-3 instantiation fall back to MINB 2 on two CTAs per
SM.  The loop's scheduling knobs (refill threshold, partial-drain threshold, staged BVH prefix, shadow-queue order, shadow overlap) change which
warp traces which ray and when, never what a ray hits: hits are keyed by (t, gid) through atomicMin, and path state and random numbers are per
path.  So no setting may move a bit of the frame, and every ray query stays the oracle's.  The frame-shape and accumulation tests hold the
per-pixel kernels (generate, commit + accumulate, tile pack / unpack) to a plain reference at the shapes where index arithmetic goes wrong."""
import numpy as np
import pytest
from test_gpu_parity import random_rays, hits_bit_equal

pytestmark = pytest.mark.gpu

W, H, SPP = 320, 180, 4
KNOBS = ("RTXPT_TRACE_CTAS", "RTXPT_SHADE_CTAS", "RTXPT_REFILL_THRESHOLD", "RTXPT_WAIT_FLUSH", "RTXPT_SMEM_NODES", "RTXPT_SHADOW_LPT", "RTXPT_OVERLAP_SHADOW",
         "RTXPT_LANES", "RTXPT_L2_PERSIST_MB")
STRICT = pytest.mark.parametrize("strict", [False, True], ids=["fast", "strict"])


def smem_node_budget(ctas, smem_optin=227 * 1024):
    """BVH nodes the staged prefix can hold at `ctas` traversal CTAs per SM (api.cu fillParams; H100: 227 KB of opt-in shared memory per block)."""
    return (min(smem_optin, 227 * 1024 // ctas - 2048) - 1024 - 8 * 2320) // 80


# the loop's scheduling knobs at their limits; the staged prefix at one node, at the budget and far above it (capped to the budget: 1182 nodes at
# two CTAs per SM are three 32 KB bulk copies, 456 at four are two)
LOOP_SETTINGS = [{}, {"RTXPT_REFILL_THRESHOLD": 1}, {"RTXPT_REFILL_THRESHOLD": 32}, {"RTXPT_WAIT_FLUSH": 1}, {"RTXPT_WAIT_FLUSH": 33}] + \
                [{"RTXPT_TRACE_CTAS": ctas, "RTXPT_SMEM_NODES": n} for ctas in (2, 4) for n in (1, smem_node_budget(ctas), 1 << 20)]


@pytest.fixture(scope="module")
def glazed_city():
    from rtxpt_b200 import scenes, scene_builder as sb
    scene, cam = scenes.city_block(target_triangles=150000, width=W, height=H, texture_size=128, n_textures=6, n_materials=64, delta_surfaces=True)
    consts = sb.make_constants(W, H, cam, bounce_count=6, diffuse_bounce_count=6, env_enabled=True, firefly_threshold=5000.0, nested_dielectrics=1, nee=True, nee_type=2)
    return scene, cam, consts


@pytest.fixture(scope="module")
def baseline():
    """Frames of the default configuration, per library, rendered once and shared by the tests below."""
    return {}


def _context(product, monkeypatch, strict, knobs=None, flags=None, **kw):
    """A context created with exactly the knobs given (every other one unset: they are read when the context is created)."""
    from rtxpt_b200 import structs as S
    knobs = knobs or {}
    for k in KNOBS:
        if k in knobs: monkeypatch.setenv(k, str(knobs[k]))
        else: monkeypatch.delenv(k, raising=False)
    kw.setdefault("max_sub_samples_per_launch", SPP)
    return product.Context(strict=strict, flags=S.CFG_EXPORT_GUIDES if flags is None else flags, **kw)


def _reference_frames(c, city, neeat=False):
    """Three frames of 4 sub-samples (6 bounces, NEE type 2); with NEE-AT, frames 1 and 2 sample lights through the feedback of the frames before."""
    scene, cam, consts = city
    c.reset_accumulation()
    colors = []
    try:
        for f in range(3):
            consts.sampleBaseIndex = f * SPP
            consts.NEEATFeedback = 1 if (neeat and f > 0) else 0        # frame 0 leaves the guides the feedback pass reprojects with
            c.set_constants(consts)
            if consts.NEEATFeedback: c.neeat_update_begin(); c.neeat_update_end()
            c.path_trace(0, SPP, True); c.synchronize()
            colors.append(c.readback_output_color())
    finally:
        consts.NEEATFeedback = 0; consts.sampleBaseIndex = 0
    return {"accumulated": c.readback_accumulated(), "output colour": np.stack(colors)}


def _realtime_frames(c, city, neeat=False):
    """Three realtime frames (BUILD + two FILL sub-samples + merge); with NEE-AT every frame adapts on the feedback of the one before."""
    from rtxpt_b200 import scene_builder as sb
    scene, cam, consts = city
    c.set_realtime(sb.make_realtime_constants(W, H, cam, bounce_count=6, sub_samples=2))
    if neeat: c.neeat_reset()
    out = {"header": [], "stable radiance": [], "output colour": []}
    try:
        for f in range(3):
            consts.sampleBaseIndex = f; consts.NEEATFeedback = 1 if neeat else 0
            c.set_constants(consts)
            if neeat: c.neeat_update_begin()
            c.path_trace_realtime(True); c.synchronize()
            g = c.readback_realtime()
            out["header"].append(g["header"]); out["stable radiance"].append(g["stable_radiance"]); out["output colour"].append(c.readback_output_color())
    finally:
        consts.NEEATFeedback = 0; consts.sampleBaseIndex = 0
    return {k: np.stack(v) for k, v in out.items()}


def _all_frames(c, city):
    """The four frame kinds that together launch every non-null entry of kTraceKernels: reference (Closest, Shadow), reference with NEE-AT
    (ShadowNeeat), realtime (ClosestRealtime, ShadowRealtime), realtime with NEE-AT (ShadowRealtimeNeeat)."""
    from rtxpt_b200 import scene_builder as sb
    scene, cam, consts = city
    c.upload_scene(scene); c.set_view(sb.world_to_clip(cam))
    frames = {"reference": _reference_frames(c, city)}
    st = c.stats()
    stats = dict(scatter=st.scatterRays, shadow=st.shadowRays, nodes=st.traversalNodeVisits, tris=st.traversalTriTests,
                 shadow_nodes=st.shadowNodeVisits, shadow_tris=st.shadowTriTests, bvh_nodes=st.bvhNodeCount)
    frames["reference, NEE-AT"] = _reference_frames(c, city, neeat=True)
    frames["realtime"] = _realtime_frames(c, city)
    frames["realtime, NEE-AT"] = _realtime_frames(c, city, neeat=True)
    return frames, stats


def _default_frames(product, monkeypatch, baseline, city, strict):
    if strict not in baseline:
        c = _context(product, monkeypatch, strict)
        try:
            baseline[strict] = _all_frames(c, city)
        finally:
            c.close()
    return baseline[strict]


def _same(a, b, what):
    """Every image of every frame kind word for word."""
    for kind in b:
        for name in b[kind]:
            x, y = np.ascontiguousarray(a[kind][name]), np.ascontiguousarray(b[kind][name])
            assert x.shape == y.shape, (what, kind, name)
            xw, yw = x.view(np.uint8).reshape(x.shape[:-1] + (-1,)), y.view(np.uint8).reshape(y.shape[:-1] + (-1,))
            assert np.array_equal(xw, yw), (what, kind, name, int((xw != yw).any(-1).sum()))


def _knob_text(knobs):
    return ", ".join("%s=%s" % kv for kv in knobs.items()) or "defaults"


@STRICT
def test_every_launch_table_entry_renders_the_default_frame(product, oracle, monkeypatch, glazed_city, baseline, strict):
    """RTXPT_TRACE_CTAS 2 / 3 / 4 x RTXPT_SHADE_CTAS 3 / 4 / 5: the MINB-2, -3 and -4 instantiations of every trace kind, and the MINB-2 fallback of the
    realtime and NEE-AT shadow kinds, render the default configuration's frames bit for bit."""
    from rtxpt_b200.imageio import per_pixel_l2
    base, base_stats = _default_frames(product, monkeypatch, baseline, glazed_city, strict)
    acc = base["reference"]["accumulated"]
    assert np.isfinite(acc).all() and acc[..., :3].mean() > 1e-3
    assert base_stats["nodes"] == 0 and base_stats["shadow_nodes"] == 0          # the default kernels count nothing
    for trace_ctas in (2, 3, 4):
        for shade_ctas in (3, 4, 5):
            if (trace_ctas, shade_ctas) == (4, 4): continue                       # the defaults
            knobs = {"RTXPT_TRACE_CTAS": trace_ctas, "RTXPT_SHADE_CTAS": shade_ctas}
            c = _context(product, monkeypatch, strict, knobs)
            try:
                frames, _ = _all_frames(c, glazed_city)
            finally:
                c.close()
            _same(frames, base, _knob_text(knobs))
    if strict:
        # the IEEE build's reference frames against the oracle on a window of the frame: 12 sub-samples in three frames, same seeds.  The city is
        # textured, and the texture units' filter weights differ from the oracle's in the last bits, so after 12 sub-samples through textured
        # vertices almost no pixel keeps every bit (H100: 0.1 %); what holds is test_cornell_c1_image_parity's largest difference and, one decade
        # above the measured 3e-7, its per-pixel L2
        scene, cam, consts = glazed_city
        rect = (144, 74, 176, 106)
        o = oracle.Oracle(scene); ref = None; n = 0
        try:
            for f in range(3):
                consts.sampleBaseIndex = f * SPP; o.set_constants(consts)
                ref, n = o.render(0, SPP, accum=ref, accum_count=n, rect=rect)[:2]
        finally:
            consts.sampleBaseIndex = 0; o.close()
        x0, y0, x1, y1 = rect
        a, b = acc[y0:y1, x0:x1], ref[y0:y1, x0:x1]
        d = np.abs(a[..., :3] - b[..., :3])
        same = float((d.max(-1) == 0).mean())
        print("glazed city window, strict build vs oracle: %.4f of pixels bit-identical, max |d| %.3g, per-pixel L2 %.3g" % (same, d.max(), per_pixel_l2(a, b)))
        assert n == 3 * SPP and b[..., :3].mean() > 1e-3                          # the window is not sky
        assert d.max() < 2e-2 and per_pixel_l2(a, b) < 3e-6


@STRICT
def test_step_counting_kernels_render_the_default_frame(product, monkeypatch, glazed_city, baseline, strict):
    """RTXPT_CFG_COUNT_TRAVERSAL_STEPS swaps in the instrumented closest-hit and shadow kernels (bench.py's roofline counts): same frames, and counts
    that fit the rays traced.  The counts themselves may differ from run to run (a lane's bestT is refreshed when its triangle tests drain)."""
    from rtxpt_b200 import structs as S
    base, _ = _default_frames(product, monkeypatch, baseline, glazed_city, strict)
    c = _context(product, monkeypatch, strict, flags=S.CFG_EXPORT_GUIDES | S.CFG_COUNT_TRAVERSAL_STEPS)
    try:
        frames, st = _all_frames(c, glazed_city)
    finally:
        c.close()
    _same(frames, base, "RTXPT_CFG_COUNT_TRAVERSAL_STEPS")
    assert st["scatter"] > 0 and st["shadow"] > 0
    assert st["nodes"] >= st["scatter"] and st["shadow_nodes"] >= st["shadow"], st           # every ray visits the root at least
    assert st["tris"] > 0 and st["shadow_tris"] > 0, st
    assert st["nodes"] <= st["scatter"] * st["bvh_nodes"] and st["shadow_nodes"] <= st["shadow"] * st["bvh_nodes"], st     # no node twice per ray


@pytest.fixture(scope="module")
def query_sets(oracle, cornell, small_city):
    """test_ray_queries_bit_exact's three query sets per scene, with the oracle's answers: random rays, bounded segments (any-hit), rays aimed at vertices."""
    sets = {}
    for which, (scene, cam) in (("cornell", cornell), ("city", small_city)):
        rng = np.random.default_rng(13)
        lo, hi = ([0.1, 0.1, -4.0], [5.4, 5.4, 5.4]) if which == "cornell" else ([-110, 0.1, -110], [110, 45, 110])
        rays = random_rays(rng, 300000, lo, hi)
        bounded = rays.copy(); bounded[:, 7] = rng.uniform(0.5, 40.0, len(rays)).astype(np.float32)
        g = scene.geometries[0]
        vb = np.ctypeslib.as_array((np.ctypeslib.ctypes.c_float * (g.numVertices * 3)).from_address(scene.buffers[g.vertexBufferIndex].data + g.positionOffset)).reshape(-1, 3)
        tgt = vb[rng.integers(0, len(vb), 20000)]
        org = np.tile(np.array([[2.7, 2.7, -3.0]] if which == "cornell" else [[3.0, 60.0, -5.0]], np.float32), (len(tgt), 1))
        edge = np.concatenate([org, np.zeros((len(tgt), 1), np.float32), (tgt - org).astype(np.float32), np.full((len(tgt), 1), 1e15, np.float32)], 1).astype(np.float32)
        o = oracle.Oracle(scene)
        sets[which] = (scene, rays, o.trace_rays(rays), bounded, o.trace_rays(bounded, any_hit=True), edge, o.trace_rays(edge))
        o.close()
    return sets


@STRICT
def test_ray_queries_match_the_oracle_at_every_loop_setting(product, monkeypatch, query_sets, strict):
    """The persistent loop's exit, refill and partial-drain rules at their limits (refill threshold 1 and 32, partial drain at 1 waiting lane or only
    when no lane traverses) and the staged BVH prefix up to its multi-chunk copy: closest hits stay the oracle's bit for bit and occlusion matches,
    also for launches of 0, 1, 31, 33 and 1000 rays, where warps run partial and the fetch cursor is exhausted at once."""
    for knobs in LOOP_SETTINGS:
        what = _knob_text(knobs)
        c = _context(product, monkeypatch, strict, knobs, flags=0)
        try:
            for which, (scene, rays, closest, bounded, occluded, edge, edge_hits) in query_sets.items():
                c.upload_scene(scene)
                assert hits_bit_equal(c.trace_rays(rays), closest).all(), (what, which, "random rays")
                assert np.array_equal(c.trace_rays(bounded, any_hit=True)["t"] >= 0, occluded["t"] >= 0), (what, which, "any-hit")
                assert hits_bit_equal(c.trace_rays(edge), edge_hits).all(), (what, which, "rays at vertices")
                for n in (0, 1, 31, 33, 1000):
                    a, b = c.trace_rays(rays[:n]), c.trace_rays(bounded[:n], any_hit=True)
                    assert len(a) == len(b) == n, (what, which, n)
                    assert hits_bit_equal(a, closest[:n]).all(), (what, which, n, "closest")
                    assert np.array_equal(b["t"] >= 0, occluded["t"][:n] >= 0), (what, which, n, "any-hit")
        finally:
            c.close()


@STRICT
def test_reference_frame_does_not_depend_on_loop_settings(product, monkeypatch, glazed_city, baseline, strict):
    """The reference frames of the launch-table test under every loop setting above, each combined in turn with one of the four combinations of
    RTXPT_SHADOW_LPT (0: every shadow record in one queue, in reverse order) and RTXPT_OVERLAP_SHADOW (0: shadow rays on the closest-hit stream)."""
    from rtxpt_b200 import scene_builder as sb
    base, _ = _default_frames(product, monkeypatch, baseline, glazed_city, strict)
    scene, cam, consts = glazed_city
    orders = [{}, {"RTXPT_SHADOW_LPT": 0}, {"RTXPT_OVERLAP_SHADOW": 0}, {"RTXPT_SHADOW_LPT": 0, "RTXPT_OVERLAP_SHADOW": 0}]
    for i, loop in enumerate(LOOP_SETTINGS):
        knobs = dict(loop, **orders[(i + 1) % len(orders)])            # the first setting (defaults) gets LPT off
        c = _context(product, monkeypatch, strict, knobs)
        try:
            c.upload_scene(scene); c.set_view(sb.world_to_clip(cam))
            frames = {"reference": _reference_frames(c, glazed_city)}
        finally:
            c.close()
        _same(frames, {"reference": base["reference"]}, _knob_text(knobs))


def _cornell_constants(w, h, **kw):
    from rtxpt_b200 import scenes, scene_builder as sb
    return sb.make_constants(w, h, scenes.cornell_box(w, h)[1], **kw)


@STRICT
def test_frame_shapes(product, oracle, monkeypatch, cornell, strict):
    """Frames smaller than a warp, pixel counts that are no multiple of 32 or 256, widths and heights that leave a ragged last 64 x 64 tile, and the
    limits set_constants accepts (65535 wide, 1 tall and the reverse): a sane frame, one path per pixel and sub-sample, and in the IEEE build the
    oracle's ray counts and, on almost every pixel, its bits (test_cornell_c1_image_parity's bounds)."""
    from rtxpt_b200.imageio import per_pixel_l2
    scene, _ = cornell
    c = _context(product, monkeypatch, strict, flags=0)
    o = oracle.Oracle(scene)
    try:
        c.upload_scene(scene)
        for w, h in ((1, 1), (7, 5), (33, 17), (200, 130), (65535, 1), (1, 4097)):
            consts = _cornell_constants(w, h, bounce_count=2, diffuse_bounce_count=2)
            c.set_constants(consts); c.reset_accumulation()
            c.path_trace(0, 1); img = c.readback_accumulated(); st = c.stats()
            assert img.shape == (h, w, 4) and np.isfinite(img).all() and (img[..., :3] >= 0).all() and (img[..., 3] == 1).all(), (w, h)
            assert st.paths == w * h and st.accumulatedSamples == 1, (w, h, st.paths)
            o.set_constants(consts)
            acc, n, _, _, ost = o.render(0, 1)
            d = np.abs(img[..., :3] - acc[..., :3])
            if strict:
                assert (st.scatterRays, st.shadowRays) == (ost.scatterRays, ost.shadowRays), (w, h)
                # almost every pixel bit-identical (0.5 %, and on the frames of a few hundred pixels or fewer, two pixels: libdevice vs glibc sin / cos)
                assert (d.max(-1) != 0).sum() <= max(2, 0.005 * w * h), (w, h, int((d.max(-1) != 0).sum()))
                assert d.max() < 2e-2 and per_pixel_l2(img, acc) < 1e-7, (w, h)
            # three more sub-samples in one launch: path slot = sub-sample * pixel count + pixel, with pixel counts that split warps
            c.path_trace(1, 3); more = c.readback_accumulated(); st = c.stats()
            assert st.paths == 3 * w * h and st.accumulatedSamples == 4 and np.isfinite(more).all() and (more[..., 3] == 1).all(), (w, h)
            acc, n, _, _, ost = o.render(1, 3, accum=acc, accum_count=n)
            if strict:
                assert (st.scatterRays, st.shadowRays) == (ost.scatterRays, ost.shadowRays) and per_pixel_l2(more, acc) < 1e-6, (w, h)
    finally:
        c.close(); o.close()


@pytest.mark.parametrize("w,h,world", [(64, 64, 4), (200, 130, 3)])
@STRICT
def test_tile_partitions_reassemble_the_frame(product, monkeypatch, cornell, w, h, world, strict):
    """Ranks of an interleaved 64 x 64 tile partition, ranks that own no pixel at all (64 x 64 over four ranks) and ranks of unequal size (200 x 130 over
    three): each renders its tiles, pack_owned / unpack_all reassemble the single-context frame bit for bit, and every call of an empty rank succeeds."""
    import torch
    scene, _ = cornell
    consts = _cornell_constants(w, h)

    def render(c):
        c.upload_scene(scene); c.set_constants(consts); c.path_trace(0, SPP); c.synchronize()
        return c.readback_accumulated()
    one = _context(product, monkeypatch, strict, flags=0)
    try:
        full = render(one)
    finally:
        one.close()
    parts = [_context(product, monkeypatch, strict, flags=0, tile_rank=r, tile_world=world, tile_size=64) for r in range(world)]
    try:
        images = [render(p) for p in parts]
        owned = [p.tile_layout() for p in parts]
        assert sum(n for n, _ in owned) == w * h and len({padded for _, padded in owned}) == 1
        assert [p.stats().paths for p in parts] == [n * SPP for n, _ in owned]
        if w * h <= 64 * 64: assert [n for n, _ in owned[1:]] == [0] * (world - 1)
        ty, tx = np.meshgrid(np.arange(h) // 64, np.arange(w) // 64, indexing="ij")
        owner = (ty * ((w + 63) // 64) + tx) % world
        for r, img in enumerate(images):
            assert np.array_equal(img[owner == r], full[owner == r]), r
        padded = owned[0][1]
        gathered = torch.zeros((world * padded, 4), dtype=torch.float32, device="cuda")
        for r, p in enumerate(parts):
            p.pack_owned(gathered[r * padded:(r + 1) * padded].data_ptr()); p.synchronize()
        for p in parts:
            p.unpack_all(gathered.data_ptr()); p.synchronize()
            assert np.array_equal(p.readback_accumulated().view(np.uint32), full.view(np.uint32))
    finally:
        for p in parts:
            p.close()


def _ulps(a, b):
    """Distance in units in the last place between float32 arrays of one sign."""
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@STRICT
def test_accumulation_replays_the_running_mean(product, monkeypatch, cornell, strict):
    """k_commit_accumulate against a plain replay: 300 launches of one sub-sample each into a 37 x 23 frame.  The output colour (RGBA16F) holds each
    launch's sample, the running mean is lerp(prev, sample, 1 / (n + 1)) with the first sample taken as it is.  The IEEE build is the float32 replay
    bit for bit.  In the default build (FMA, approximate reciprocal) every launch's step is within 2 ulp of the step replayed from the buffer it
    found (H100 SXM, 700 W: 1 ulp); over the 300 launches those one-step differences add up to 4 ulp from the replay, held here to 8.  Both builds
    are within 1e-5 of the float64 mean."""
    scene, _ = cornell
    w, h, launches = 37, 23, 300
    consts = _cornell_constants(w, h, bounce_count=3, diffuse_bounce_count=3)
    c = _context(product, monkeypatch, strict, flags=0, max_sub_samples_per_launch=1)
    try:
        c.upload_scene(scene); c.set_constants(consts)
        def lerp(prev, s, n):
            blend = np.float32(1.0) / np.float32(n + 1)
            return s if blend >= 1 else (prev + (s - prev) * blend).astype(np.float32)
        replay = acc = np.zeros((h, w, 4), np.float32); total = np.zeros((h, w, 3), np.float64)
        worst = worst_step = 0
        for i in range(launches):
            prev = acc
            c.path_trace(i, 1); sample = c.readback_output_color().astype(np.float32); acc = c.readback_accumulated()
            assert (sample[..., 3] == 1).all() and c.stats().accumulatedSamples == i + 1
            s = sample.copy(); s[..., 3] = 1.0
            replay = lerp(replay, s, i)
            total += sample[..., :3]
            if i == 0: assert np.array_equal(acc, s)                          # the first sample overwrites whatever the buffer held
            if strict: assert np.array_equal(acc.view(np.uint32), replay.view(np.uint32)), (i, int((acc != replay).any(-1).sum()))
            else:
                worst_step = max(worst_step, int(_ulps(acc, lerp(prev, s, i)).max()))        # this launch's step from the buffer it found
                worst = max(worst, int(_ulps(acc, replay).max()))
        mean = total / launches
        assert (np.abs(acc[..., :3] - mean) <= 1e-5 * np.abs(mean)).all(), float((np.abs(acc[..., :3] - mean) / np.maximum(np.abs(mean), 1e-30)).max())
        assert mean.mean() > 1e-3 and (mean.max(-1) > 0).mean() > 0.5          # at this aspect ratio the frame's left and right thirds look past the box
        print("running mean, %s build: at most %d ulp from the float32 replay over %d launches, %d ulp in one launch" % ("strict" if strict else "fast", worst, launches, worst_step))
        assert worst_step <= 2 and worst <= 8, (worst_step, worst)
        # a launch without accumulation only writes the output colour; reset_accumulation restarts the count and the next sample overwrites
        c.path_trace(launches, 1, accumulate=False)
        assert np.array_equal(c.readback_accumulated(), acc) and c.stats().accumulatedSamples == launches
        c.reset_accumulation(); c.path_trace(launches + 1, 1)
        s = c.readback_output_color().astype(np.float32); s[..., 3] = 1.0
        assert c.stats().accumulatedSamples == 1 and np.array_equal(c.readback_accumulated(), s)
    finally:
        c.close()
