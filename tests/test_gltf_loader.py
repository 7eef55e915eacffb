"""The library's host-side glTF loader (rtxpt_b200/csrc/gltf_loader.cpp) against the table builder of rtxpt_b200/scene_builder.py: the same
scene authored in numpy and written out as glTF must come back as the same GPU tables, byte for byte.  CPU only."""
import ctypes as C
import os
import numpy as np
import pytest
import gltf_export


def _bytes(ptr, n):
    return bytes((C.c_uint8 * n).from_address(C.addressof(ptr.contents) if hasattr(ptr, "contents") else ptr)) if n else b""


def _table(ptr, count, typ):
    return bytes((C.c_uint8 * (count * C.sizeof(typ))).from_address(C.addressof(ptr.contents))) if count else b""


def _compare_scenes(py_scene, gl_scene, emissive_rtol=0.0):
    from rtxpt_b200 import structs as S
    a, b = py_scene.desc, gl_scene.desc
    assert (a.instanceCount, a.geometryCount, a.subInstanceCount, a.bufferCount, a.textureCount, a.lightCount) == \
           (b.instanceCount, b.geometryCount, b.subInstanceCount, b.bufferCount, b.textureCount, b.lightCount)
    assert b.materialCount == a.materialCount + 1                  # + the glTF default material
    assert _table(a.instances, a.instanceCount, S.InstanceData) == _table(b.instances, b.instanceCount, S.InstanceData)
    assert _table(a.geometries, a.geometryCount, S.GeometryData) == _table(b.geometries, b.geometryCount, S.GeometryData)
    assert _table(a.subInstances, a.subInstanceCount, S.SubInstanceData) == _table(b.subInstances, b.subInstanceCount, S.SubInstanceData)
    for i in range(a.materialCount):
        ma, mb = a.materials[i], b.materials[i]
        for name, _ in S.MaterialData._fields_:
            va, vb = getattr(ma, name), getattr(mb, name)
            if name == "EmissiveColor":
                assert np.allclose(list(va), list(vb), rtol=emissive_rtol, atol=0), (i, name, list(va), list(vb))
            elif hasattr(va, "__len__"): assert list(va) == list(vb), (i, name, list(va), list(vb))
            else: assert va == vb, (i, name, va, vb)
    for i in range(a.bufferCount):
        assert a.buffers[i].sizeBytes == b.buffers[i].sizeBytes, i
        n = a.buffers[i].sizeBytes
        ba = bytes((C.c_uint8 * n).from_address(a.buffers[i].data)); bb = bytes((C.c_uint8 * n).from_address(b.buffers[i].data))
        if ba != bb:
            d = np.nonzero(np.frombuffer(ba, np.uint8) != np.frombuffer(bb, np.uint8))[0]
            raise AssertionError("buffer %d differs at %d bytes, first offsets %s of %d" % (i, len(d), d[:8], n))
    for i in range(a.textureCount):
        ta, tb = a.textures[i], b.textures[i]
        assert (ta.width, ta.height, ta.mipLevels, ta.format) == (tb.width, tb.height, tb.mipLevels, tb.format)
        for m in range(ta.mipLevels):
            n = max(1, ta.width >> m) * max(1, ta.height >> m) * 4
            assert bytes((C.c_uint8 * n).from_address(ta.mips[m])) == bytes((C.c_uint8 * n).from_address(tb.mips[m])), (i, m)
    if a.lightCount:
        la = np.frombuffer(_table(a.lights, a.lightCount, S.LightDesc), np.float32).reshape(a.lightCount, 15)
        lb = np.frombuffer(_table(b.lights, b.lightCount, S.LightDesc), np.float32).reshape(b.lightCount, 15)
        assert np.array_equal(la[:, 0].view(np.uint32), lb[:, 0].view(np.uint32))
        la, lb = la.copy(), lb.copy()
        for l in (la, lb): l[:, 4:7] /= np.linalg.norm(l[:, 4:7], axis=1, keepdims=True)      # the glTF node carries the normalised axis
        assert np.allclose(la[:, 1:14], lb[:, 1:14], rtol=2e-6, atol=1e-6)       # positions exact, axis / cone angles through double <-> degrees


def _textured_builder():
    from rtxpt_b200.scene_builder import SceneBuilder, Material, translate_scale
    from rtxpt_b200.scenes import _quad, _box, _merge
    rng = np.random.default_rng(7)
    b = SceneBuilder()
    t_base = b.add_texture(rng.integers(0, 256, (32, 16, 4), dtype=np.uint8), srgb=True)          # non-square, alpha channel used by the cutout
    t_nrm = b.add_texture(rng.integers(96, 160, (16, 16, 4), dtype=np.uint8), srgb=False)
    t_em = b.add_texture(rng.integers(0, 256, (8, 8, 4), dtype=np.uint8), srgb=True)
    m0 = b.add_material(Material(base_color=(0.8, 0.7, 0.6), roughness=0.45, metalness=0.2, base_texture=t_base, normal_texture=t_nrm, normal_scale=0.75))
    m1 = b.add_material(Material(base_color=(1, 1, 1), roughness=0.9, base_texture=t_base, alpha_test=True, alpha_cutoff=0.4))
    m2 = b.add_material(Material(base_color=(0.9, 0.95, 1.0), roughness=0.05, transmission=0.95, ior=1.45, thin_surface=False, volume_color=(0.8, 0.9, 1.0), volume_distance=2.5, nested_priority=3))
    m3 = b.add_material(Material(base_color=(0.2, 0.2, 0.2), roughness=1.0, emissive=(1.0, 0.5, 0.25), emissive_intensity=8.0, emissive_texture=t_em))
    def with_uv(g, scale=1.0):
        g = dict(g); p = np.asarray(g["positions"], np.float32); g["uvs"] = np.stack([p[:, 0] * 0.37 + p[:, 2] * 0.11, p[:, 1] * 0.29 - p[:, 2] * 0.23], 1).astype(np.float32) * np.float32(scale); return g
    ground = with_uv(_quad((-4, 0, -4), (-4, 0, 4), (4, 0, 4), (4, 0, -4), m0))
    wall = with_uv(_quad((-4, 0, 4), (-4, 3, 4), (4, 3, 4), (4, 0, 4), m1), 2.0)
    glass = _merge(_box([(-1, 0, -1), (-1, 0, 1), (1, 0, 1), (1, 0, -1)], 2.0, m2), m2)           # no uvs: zero tangents, texCoord offset absent
    lamp = with_uv(_quad((-0.5, 2.9, -0.5), (0.5, 2.9, -0.5), (0.5, 2.9, 0.5), (-0.5, 2.9, 0.5), m3))
    b.add_mesh([ground, wall]); b.add_mesh([glass]); b.add_mesh([lamp])
    b.add_instance(0); b.add_instance(1, translate_scale((0.5, 0.0, -0.25), (0.5, 1.25, 0.75))); b.add_instance(1, translate_scale((-2.0, 0.0, 1.0))); b.add_instance(2)
    b.add_point_light(position=(1.5, 2.0, -1.0), color=(1.0, 0.9, 0.8), intensity=20.0, radius=0.1)
    b.add_spot_light(position=(-2.0, 2.5, -2.0), direction=(0.4, -1.0, 0.3), color=(0.6, 0.7, 1.0), intensity=35.0, radius=0.05, inner_angle=12.0, outer_angle=30.0)
    return b


def test_cornell_gltf_matches_table_builder(product, oracle, tmp_path):
    """BASELINE.json configs[0] is a Cornell-box glTF: authored here, written as glTF, loaded by the C++ loader, rendered by the oracle."""
    from rtxpt_b200 import scenes, scene_builder as sb
    from rtxpt_b200.scene_builder import SceneBuilder
    py_scene, cam = scenes.cornell_box(64, 64)
    # re-create the builder the stand-in scene was made from (cornell_box returns the built scene)
    b = scenes.cornell_builder()
    path = gltf_export.export(b, str(tmp_path / "cornell.gltf"), camera=dict(position=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), yfov=0.66, znear=0.1, zfar=1e7))
    gl = product.GltfScene(path)
    assert gl.triangle_count == 36 and gl.desc.instanceCount == 3 and gl.desc.geometryCount == 6
    _compare_scenes(py_scene, gl, emissive_rtol=2e-7)
    c = gl.cameras[0]
    assert np.allclose(c.position[:], (2.78, 2.73, -8.0)) and np.allclose(c.direction[:], (0, 0, 1), atol=1e-6) and np.allclose(c.up[:], (0, 1, 0), atol=1e-6) and abs(c.yfov - 0.66) < 1e-6
    consts = sb.make_constants(64, 64, cam, bounce_count=2, diffuse_bounce_count=2)
    o1 = oracle.Oracle(py_scene); o1.set_constants(consts); a = o1.render(0, 1)[0]; o1.close()
    o2 = oracle.Oracle(gl); o2.set_constants(consts); b_ = o2.render(0, 1)[0]; o2.close()
    assert np.abs(a - b_).max() <= 1e-3 * max(1.0, float(a.max()))        # identical geometry; the lamp's emissive differs by one float ulp (17 * (12/17))
    gl.close()


@pytest.mark.parametrize("glb", [False, True])
def test_textured_gltf_matches_table_builder(product, tmp_path, glb):
    """Textures (PNG, sRGB / linear slots, mips), computed tangents, alpha-tested / transmissive / emissive materials, instancing with
    transforms, analytic lights: every table and every buffer byte equals what scene_builder.py produces from the same data."""
    b = _textured_builder()
    py_scene = b.build()
    path = gltf_export.export(b, str(tmp_path / ("scene.glb" if glb else "scene.gltf")), glb=glb)
    gl = product.GltfScene(path)
    _compare_scenes(py_scene, gl, emissive_rtol=2e-7)
    assert gl.triangle_count == py_scene.triangle_count
    gl.close()


def test_gltf_loader_errors(product, tmp_path):
    import json
    with pytest.raises(product.RtxptError, match="cannot open"):
        product.GltfScene(str(tmp_path / "missing.gltf"))
    bad = tmp_path / "bad.gltf"; bad.write_text("{ \"asset\": ")
    with pytest.raises(product.RtxptError, match="JSON"):
        product.GltfScene(str(bad))
    b = _textured_builder(); path = gltf_export.export(b, str(tmp_path / "s.gltf"))
    doc = json.load(open(path))
    doc2 = dict(doc); doc2["extensionsRequired"] = ["KHR_draco_mesh_compression"]; json.dump(doc2, open(tmp_path / "draco.gltf", "w"))
    with pytest.raises(product.RtxptError, match="required extension"):
        product.GltfScene(str(tmp_path / "draco.gltf"))
    doc3 = json.loads(json.dumps(doc)); doc3["accessors"][0]["sparse"] = {"count": 1}; json.dump(doc3, open(tmp_path / "sparse.gltf", "w"))
    with pytest.raises(product.RtxptError, match="sparse"):
        product.GltfScene(str(tmp_path / "sparse.gltf"))
    (tmp_path / "s_tex0.png").write_bytes(b"GIF89a not a png")                      # neither PNG nor JPEG nor DDS
    with pytest.raises(product.RtxptError, match="not a PNG"):
        product.GltfScene(path)
    (tmp_path / "s_tex0.png").write_bytes(b"\xff\xd8\xff\xe0 a JPEG signature and nothing behind it")
    with pytest.raises(product.RtxptError, match="JPEG"):
        product.GltfScene(path)


def test_host_helpers_match_python_mirror(product):
    """rtxpt_b200_bridge_camera / rtxpt_b200_default_constants (C++) against scene_builder.bridge_camera / make_constants."""
    from rtxpt_b200 import scene_builder as sb, structs as S
    L = product.load()
    f3 = lambda v: (C.c_float * 3)(*v)
    for (w, h, pos, d, up, fov, jit) in [(256, 256, (2.78, 2.73, -8.0), (0, 0, 1), (0, 1, 0), 0.66, (0.0, 0.0)), (1920, 1080, (-20, 1.8, 12), (0.7, -0.1, 0.7), (0, 1, 0), 1.04, (0.25, -0.5))]:
        out = S.CameraData()
        assert L.rtxpt_b200_bridge_camera(w, h, f3(pos), f3(d), f3(up), fov, 0.1, 1e7, 10000.0, 0.0, (C.c_float * 2)(*jit), C.byref(out)) == 0
        ref = sb.bridge_camera(w, h, pos, d, up, fov, jitter=jit)
        a = np.frombuffer(bytes(out), np.float32); b = np.frombuffer(bytes(ref), np.float32)
        assert np.allclose(a, b, rtol=3e-7, atol=0) and list(out.ViewportSize) == [w, h]
        k = S.PathTracerConstants(); assert L.rtxpt_b200_default_constants(C.byref(out), 1, C.byref(k)) == 0
        r = sb.make_constants(w, h, out, bounce_count=20, diffuse_bounce_count=2, firefly_threshold=5000.0, env_enabled=True)
        assert bytes(k) == bytes(r)


def test_cpp_host_example_without_gpu(product, tmp_path):
    """The C++ example host links against the C ABI only; without a CUDA device it must stop at create() with the no-fallback message."""
    import subprocess, torch
    if torch.cuda.is_available():
        pytest.skip("needs a machine without a GPU")
    from rtxpt_b200 import scenes
    exe = os.path.join(os.path.dirname(product.LIB_PATH), "render_gltf")
    path = gltf_export.export(scenes.cornell_builder(), str(tmp_path / "cornell.gltf"), camera=dict(position=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), yfov=0.66, znear=0.1, zfar=1e7))
    r = subprocess.run([exe, path, str(tmp_path / "o.pfm"), "32", "32", "1", "2"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "no CPU fallback" in r.stderr
    exe = os.path.join(os.path.dirname(product.LIB_PATH), "realtime_gltf")
    r = subprocess.run([exe, path, str(tmp_path / "o.ppm"), "32", "32", "2", "2"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_cpp_realtime_example_writes_a_tone_mapped_frame(product, tmp_path):
    """glTF file -> examples/realtime_gltf.cpp (NEE-AT update, stable-plane BUILD/FILL, ReBLUR, tone mapping through the C ABI only) -> PPM: the box is lit, not saturated, and the
    image differs from a flat fill."""
    import subprocess
    from rtxpt_b200 import scenes
    exe = os.path.join(os.path.dirname(product.LIB_PATH), "realtime_gltf")
    path = gltf_export.export(scenes.cornell_builder(), str(tmp_path / "cornell.gltf"), camera=dict(position=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), yfov=0.66, znear=0.1, zfar=1e7))
    out = str(tmp_path / "o.ppm")
    r = subprocess.run([exe, path, out, "128", "128", "8", "4"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f:
        assert f.readline() == b"P6\n" and f.readline() == b"128 128\n" and f.readline() == b"255\n"
        img = np.frombuffer(f.read(), np.uint8).reshape(128, 128, 3)
    assert 20 < img.mean() < 235 and img.std() > 10


@pytest.mark.gpu
def test_cpp_host_example_renders_cornell(product, oracle, tmp_path):
    """glTF file -> C++ host (examples/render_gltf.cpp) -> PFM, against the oracle rendering the table-builder scene."""
    import subprocess
    from rtxpt_b200 import scenes, scene_builder as sb
    from rtxpt_b200.imageio import per_pixel_l2
    exe = os.path.join(os.path.dirname(product.LIB_PATH), "render_gltf")
    path = gltf_export.export(scenes.cornell_builder(), str(tmp_path / "cornell.gltf"), camera=dict(position=(2.78, 2.73, -8.0), direction=(0, 0, 1), up=(0, 1, 0), yfov=0.66, znear=0.1, zfar=1e7))
    out = str(tmp_path / "o.pfm")
    r = subprocess.run([exe, path, out, "96", "96", "8", "2"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f:
        assert f.readline() == b"PF\n" and f.readline() == b"96 96\n" and f.readline() == b"-1.0\n"
        img = np.frombuffer(f.read(), np.float32).reshape(96, 96, 3)[::-1]
    scene, cam = scenes.cornell_box(96, 96)
    consts = sb.make_constants(96, 96, cam, bounce_count=2, diffuse_bounce_count=2, firefly_threshold=5000.0)
    o = oracle.Oracle(scene); acc = None; n = 0
    for base in (0, 4):
        consts.sampleBaseIndex = base; o.set_constants(consts); acc, n = o.render(0, 4, accum=acc, accum_count=n)[:2]
    o.close()
    assert per_pixel_l2(np.concatenate([img, np.ones((96, 96, 1), np.float32)], -1), acc) < 1e-4


def test_loaders_refuse_hostile_files(product, tmp_path):
    """Untrusted input: accessor offsets / strides / counts that would read outside their bufferView, a PNG whose IHDR lies about itself, JSON nested beyond any real scene,
    a DDS header claiming more mips than the image can have - each refused with a message, none crashes or over-allocates."""
    import json, struct, zlib
    b = _textured_builder(); path = gltf_export.export(b, str(tmp_path / "s.gltf")); doc = json.load(open(path))
    def load_with(mutator, name):
        d = json.loads(json.dumps(doc)); mutator(d); json.dump(d, open(tmp_path / name, "w")); return product.GltfScene(str(tmp_path / name))
    pos_acc = doc["meshes"][0]["primitives"][0]["attributes"]["POSITION"]; bv = doc["accessors"][pos_acc]["bufferView"]
    for mut, match in ((lambda d: d["accessors"][pos_acc].__setitem__("byteOffset", -16), "byteOffset"),
                       (lambda d: d["accessors"][pos_acc].__setitem__("byteOffset", 1e30), "byteOffset"),
                       (lambda d: d["bufferViews"][bv].__setitem__("byteStride", 1 << 40), "byteStride"),
                       (lambda d: d["bufferViews"][bv].__setitem__("byteStride", 4), "byteStride"),
                       (lambda d: d["bufferViews"][bv].__setitem__("byteLength", 24), "past the end of bufferView"),
                       (lambda d: d["bufferViews"][bv].__setitem__("byteOffset", 1 << 33), "byteOffset|outside buffer"),
                       (lambda d: d["accessors"][pos_acc].__setitem__("count", 1 << 30), "past the end")):
        with pytest.raises(product.RtxptError, match=match): load_with(mut, "hostile.gltf")
    # JSON nesting
    deep = tmp_path / "deep.gltf"; deep.write_text("[" * 100000)
    with pytest.raises(product.RtxptError, match="nesting"): product.GltfScene(str(deep))
    # PNG: IHDR of the wrong length; absurd dimensions
    def png(ihdr, extra_len=0):
        def chunk(t, data): return struct.pack(">I", len(data)) + t + data + struct.pack(">I", zlib.crc32(t + data) & 0xffffffff)
        return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IDAT", zlib.compress(b"\0" * 8)) + chunk(b"IEND", b"")
    tex = [n for n in os.listdir(tmp_path) if n.endswith(".png")][0]
    (tmp_path / tex).write_bytes(png(struct.pack(">II", 4, 4) + b"\x08"))                      # 9-byte IHDR
    with pytest.raises(product.RtxptError, match="IHDR"): product.GltfScene(path)
    (tmp_path / tex).write_bytes(png(struct.pack(">IIBBBBB", 1 << 30, 1 << 30, 8, 6, 0, 0, 0)))
    with pytest.raises(product.RtxptError, match="larger than"): product.GltfScene(path)
    # DDS: 2x2 RGBA8 image whose header claims 40 mips decodes as its real chain (2 levels), not 40 shifts
    from test_dds import dds_dx10
    data = bytearray(dds_dx10("RGBA8", 2, 2, bytes(16) + bytes(4), mips=2)); data[28:32] = struct.pack("<I", 40)
    rgba, mips, _ = product.decode_dds(bytes(data)); assert mips == 2 and rgba.shape[:2] == (2, 2)
