"""DDS / block-compression decoding of the host loader against an independent decoder (Pillow's DDS plugin), block by block on random data
(random bits exercise every BC7 mode, partition, rotation and index-selector), plus the container variants (legacy FourCC, DX10 header, mips,
non-multiple-of-4 sizes).  Host only - no GPU, no oracle."""
import io
import struct

import numpy as np
import pytest

from rtxpt_b200 import lib as L

PIL = pytest.importorskip("PIL.Image")

DXGI = {"BC1": 71, "BC2": 74, "BC3": 77, "BC4": 80, "BC5": 83, "BC7": 98, "BC7_SRGB": 99, "RGBA8": 28, "BGRA8": 87}
BLOCK_BYTES = {"BC1": 8, "BC2": 16, "BC3": 16, "BC4": 8, "BC5": 16, "BC7": 16, "BC7_SRGB": 16}


def dds_dx10(fmt, width, height, payload, mips=1):
    hdr = struct.pack("<4sIIIIIII44xIIIIIIIIIIII4x", b"DDS ", 124, 0x1007 | (0x20000 if mips > 1 else 0), height, width, 0, 0, mips,
                      32, 0x4, int.from_bytes(b"DX10", "little"), 0, 0, 0, 0, 0, 0x1000, 0, 0, 0)
    assert len(hdr) == 128, len(hdr)
    return hdr + struct.pack("<IIIII", DXGI[fmt], 3, 0, 1, 0) + payload


def dds_fourcc(fourcc, width, height, payload):
    hdr = struct.pack("<4sIIIIIII44xIIIIIIIIIIII4x", b"DDS ", 124, 0x1007, height, width, 0, 0, 1, 32, 0x4, int.from_bytes(fourcc, "little"), 0, 0, 0, 0, 0, 0x1000, 0, 0, 0)
    return hdr + payload


def pil_decode(file_bytes):
    im = PIL.open(io.BytesIO(file_bytes)); im.load()
    return im.mode, np.asarray(im)


def compare(fmt, ours, mode, theirs):
    if fmt in ("BC4",):
        assert mode == "L"; np.testing.assert_array_equal(ours[..., 0], theirs); assert (ours[..., 3] == 255).all()
    elif fmt == "BC5":
        assert mode == "RGB"; np.testing.assert_array_equal(ours[..., :2], theirs[..., :2])
    elif mode == "RGB":
        np.testing.assert_array_equal(ours[..., :3], theirs); assert (ours[..., 3] == 255).all()
    else:
        assert mode == "RGBA"; np.testing.assert_array_equal(ours, theirs)


@pytest.mark.parametrize("fmt", ["BC1", "BC2", "BC3", "BC4", "BC5", "BC7"])
def test_random_blocks_match_pillow(fmt):
    rng = np.random.default_rng(hash(fmt) & 0xFFFF); W, H = 256, 128
    payload = rng.integers(0, 256, (W // 4) * (H // 4) * BLOCK_BYTES[fmt], dtype=np.uint8)
    if fmt == "BC7":          # spread the modes evenly: random bytes alone make mode 0 half of all blocks and mode 7 under 1 %
        blocks = payload.reshape(-1, 16); modes = rng.integers(0, 8, len(blocks))
        blocks[:, 0] = (blocks[:, 0] & ~((1 << (modes + 1)) - 1).astype(np.uint8)) | (1 << modes).astype(np.uint8)
    data = dds_dx10(fmt, W, H, payload.tobytes())
    ours, mips, srgb = L.decode_dds(data)
    assert ours.shape == (H, W, 4) and mips == 1 and not srgb
    mode, theirs = pil_decode(data)
    compare(fmt, ours, mode, theirs)


def test_bc7_every_mode_is_covered_and_reserved_mode_is_transparent():
    rng = np.random.default_rng(7)
    for mode in range(8):
        blocks = rng.integers(0, 256, (64, 16), dtype=np.uint8)
        blocks[:, 0] = (blocks[:, 0] & ~np.uint8((1 << (mode + 1)) - 1)) | np.uint8(1 << mode)
        data = dds_dx10("BC7", 32, 32, blocks.tobytes())
        ours, _, _ = L.decode_dds(data); m, theirs = pil_decode(data)
        compare("BC7", ours, m, theirs)
        if mode < 4: assert (ours[..., 3] == 255).all()       # modes 0-3 carry no alpha
    zero = dds_dx10("BC7", 4, 4, bytes(16))
    ours, _, _ = L.decode_dds(zero); assert (ours == 0).all()


def test_container_variants():
    rng = np.random.default_rng(3)
    # legacy FourCC headers decode like their DX10 equivalents
    for fourcc, fmt in ((b"DXT1", "BC1"), (b"DXT3", "BC2"), (b"DXT5", "BC3"), (b"ATI1", "BC4"), (b"ATI2", "BC5")):
        payload = rng.integers(0, 256, 4 * 4 * BLOCK_BYTES[fmt], dtype=np.uint8).tobytes()
        a, _, _ = L.decode_dds(dds_fourcc(fourcc, 16, 16, payload)); b, _, _ = L.decode_dds(dds_dx10(fmt, 16, 16, payload))
        np.testing.assert_array_equal(a, b)
    # sRGB flag
    _, _, srgb = L.decode_dds(dds_dx10("BC7_SRGB", 4, 4, bytes([0x40] + [0] * 15))); assert srgb
    # mip chain + sizes that are not multiples of four: 10x6 -> 5x3 -> 2x1 -> 1x1
    sizes = [(10, 6), (5, 3), (2, 1), (1, 1)]; payload = b""; chunks = []
    for (w, h) in sizes:
        c = rng.integers(0, 256, ((w + 3) // 4) * ((h + 3) // 4) * 16, dtype=np.uint8).tobytes(); chunks.append(c); payload += c
    data = dds_dx10("BC3", 10, 6, payload, mips=4)
    for m, (w, h) in enumerate(sizes):
        img, n, _ = L.decode_dds(data, mip=m); assert n == 4 and img.shape == (h, w, 4)
        full, _, _ = L.decode_dds(dds_dx10("BC3", (w + 3) // 4 * 4, (h + 3) // 4 * 4, chunks[m]))
        np.testing.assert_array_equal(img, full[:h, :w])
    # uncompressed
    px = rng.integers(0, 256, (5, 7, 4), dtype=np.uint8)
    a, _, _ = L.decode_dds(dds_dx10("RGBA8", 7, 5, px.tobytes())); np.testing.assert_array_equal(a, px)
    b, _, _ = L.decode_dds(dds_dx10("BGRA8", 7, 5, px.tobytes())); np.testing.assert_array_equal(b, px[..., [2, 1, 0, 3]])


def test_errors_are_reported():
    with pytest.raises(L.RtxptError, match="not a DDS"): L.decode_dds(b"PNG!" + bytes(200))
    with pytest.raises(L.RtxptError, match="truncated"): L.decode_dds(dds_dx10("BC7", 64, 64, bytes(16)))
    bc6 = bytearray(dds_dx10("BC7", 4, 4, bytes(16))); bc6[128:132] = struct.pack("<I", 95)
    with pytest.raises(L.RtxptError, match="BC6H"): L.decode_dds(bytes(bc6))          # an HDR format is not a material texture: rtxpt_b200_load_dds_hdr reads it
    with pytest.raises(L.RtxptError, match="not an HDR format"): L.load_dds_hdr(dds_dx10("BC7", 4, 4, bytes(16)))


# ---- HDR DDS: BC6H (the reference's *_cube_bc6u.dds environment maps), RGBA16F, RGBA32F ------------------------------------------------------------------------------------
def _hdr_dx10(dxgi, width, height, payload, mips=1, cube=False, array=1):
    hdr = struct.pack("<4sIIIIIII44xIIIIIIIIIIII4x", b"DDS ", 124, 0x1007 | (0x20000 if mips > 1 else 0), height, width, 0, 0, mips,
                      32, 0x4, int.from_bytes(b"DX10", "little"), 0, 0, 0, 0, 0, 0x1000, 0xFE00 if cube else 0, 0, 0)
    return hdr + struct.pack("<IIIII", dxgi, 3, 0x4 if cube else 0, array, 0) + payload


def _pillow_bc6_bytes(rgba):
    """Pillow decodes BC6H to 8-bit RGB: clamp to [0, 1], times 255, truncated."""
    v = np.nan_to_num(rgba[..., :3].astype(np.float64), nan=0.0, posinf=2.0, neginf=-1.0)
    return (np.clip(v, 0.0, 1.0) * 255.0).astype(np.uint8)


@pytest.mark.parametrize("signed", [False, True])
def test_bc6h_random_blocks_match_pillow(signed):
    """Random 128-bit blocks exercise all 14 modes, every partition and both index widths; Pillow's decoder is the independent check (8-bit after clamping: about a quarter
    of the texels land strictly inside (0, 1) and compare with 1/255 resolution; the rest checks zero / saturated agreement, i.e. the mode and endpoint plumbing)."""
    rng = np.random.default_rng(95 + signed); W, H = 256, 256
    blocks = rng.integers(0, 256, ((W // 4) * (H // 4), 16), dtype=np.uint8)
    # spread the modes evenly (random bits make the two 2-bit modes half of all blocks) and keep the exponent field of some endpoints small so that more texels fall inside (0, 1)
    pool = [0x00, 0x01, 0x02, 0x06, 0x0A, 0x0E, 0x12, 0x16, 0x1A, 0x1E, 0x03, 0x07, 0x0B, 0x0F]
    if signed: pool = [0x1E, 0x03, 0x0F]      # SF16: Pillow and this decoder (which follows the D3D11.3 decode: wrap to the endpoint precision, then sign-extend) disagree on the transformed
                                              # modes below 16 bits; the reference's environment maps are all UF16 ("bc6u"), so the signed path is held to the modes both decoders agree on
    modes = np.array(pool, np.uint8)[rng.integers(0, len(pool), len(blocks))]
    two = modes < 2
    blocks[:, 0] = np.where(two, (blocks[:, 0] & 0xFC) | modes, (blocks[:, 0] & 0xE0) | modes)
    data = _hdr_dx10(96 if signed else 95, W, H, blocks.tobytes())
    ours, mips = L.load_dds_hdr(data)
    assert ours.shape == (1, H, W, 4) and mips == 1 and (ours[..., 3] == 1).all()
    im = PIL.open(io.BytesIO(data)); im.load(); theirs = np.asarray(im)
    assert im.mode == "RGB" and theirs.shape == (H, W, 3)
    mine = _pillow_bc6_bytes(ours[0])
    diff = np.abs(mine.astype(int) - theirs.astype(int))
    assert (diff <= 1).mean() > 0.9999, ((diff > 1).mean(), np.unique(modes[(diff.reshape(H // 4, 4, W // 4, 4, 3).max((1, 3, 4)) > 1).reshape(-1)]))
    inside = (theirs > 0) & (theirs < 255)
    assert inside.mean() > 0.08                                                  # the comparison is not only zeros and saturated texels
    if not signed: assert (ours[0][..., :3] >= 0).all()
    else: assert (ours[0][..., :3] < 0).any()
    assert np.isfinite(ours).all()                                               # BC6H cannot encode Inf / NaN (the largest code is 0x7BFF = 65504)


def test_bc6h_reserved_modes_decode_to_zero_and_known_block():
    for m in (0x13, 0x17, 0x1B, 0x1F):
        blk = bytearray(np.random.default_rng(m).integers(0, 256, 16, dtype=np.uint8).tobytes()); blk[0] = (blk[0] & 0xE0) | m
        out, _ = L.load_dds_hdr(_hdr_dx10(95, 4, 4, bytes(blk))); assert (out[..., :3] == 0).all()
    # mode 11 (10.10, one region, no transform): endpoints A = B = (1023, 0, 512) -> unquantised 0xFFFF, 0, ((512 << 15) + 0x4000) >> 9 = 32800 -> finish (x * 31) >> 6
    bits = 0x03 | (1023 << 5) | (0 << 15) | (512 << 25) | (1023 << 35) | (0 << 45) | (512 << 55)
    out, _ = L.load_dds_hdr(_hdr_dx10(95, 4, 4, bits.to_bytes(16, "little")))
    want = np.array([(0xFFFF * 31) >> 6, 0, (32800 * 31) >> 6], np.uint16).view(np.float16).astype(np.float32)
    assert np.array_equal(out[0, :, :, :3], np.broadcast_to(want, (4, 4, 3)))


def test_hdr_float_formats_and_cubes():
    rng = np.random.default_rng(5)
    px = rng.random((6, 8, 8, 4), dtype=np.float32) * 10
    mip1 = rng.random((6, 4, 4, 4), dtype=np.float32)
    payload = b"".join(px[f].tobytes() + mip1[f].tobytes() for f in range(6))                 # per face: the whole mip chain
    out, mips = L.load_dds_hdr(_hdr_dx10(2, 8, 8, payload, mips=2, cube=True)); assert mips == 2 and np.array_equal(out, px)
    h = px.astype(np.float16)
    out, _ = L.load_dds_hdr(_hdr_dx10(10, 8, 8, b"".join(h[f].tobytes() for f in range(6)), cube=True)); assert np.array_equal(out, h.astype(np.float32))
    blocks = rng.integers(0, 256, (6, 4, 16), dtype=np.uint8)
    cube, _ = L.load_dds_hdr(_hdr_dx10(95, 8, 8, blocks.tobytes(), cube=True)); assert cube.shape == (6, 8, 8, 4)
    for f in range(6):
        one, _ = L.load_dds_hdr(_hdr_dx10(95, 8, 8, blocks[f].tobytes())); assert np.array_equal(cube[f], one[0])
    with pytest.raises(L.RtxptError, match="truncated"): L.load_dds_hdr(_hdr_dx10(95, 8, 8, bytes(16 * 3)))


def _texture_pixels(desc, slot, mip=0):
    import ctypes as C
    t = desc.textures[slot]; w, h = max(1, t.width >> mip), max(1, t.height >> mip)
    return np.frombuffer(C.string_at(t.mips[mip], w * h * 4), np.uint8).reshape(h, w, 4).copy()


def test_dds_textures_through_the_scene_loaders(tmp_path):
    """The three ways a DDS reaches a material in the reference: a .dds sibling of a glTF PNG (GltfImporter.cpp:786-796), an MSFT_texture_dds
    image (GltfImporter.cpp:853-860) and the texture paths of .material.json files, relative to the media folder with the same .png -> .dds
    swap (MaterialsBaker.cpp:159-195)."""
    import json, sys, os
    sys.path.insert(0, os.path.dirname(__file__))
    import gltf_export
    from test_gltf_loader import _textured_builder
    from rtxpt_b200 import structs as S
    rng = np.random.default_rng(11)
    media = tmp_path / "Assets"; (media / "Models").mkdir(parents=True); (media / "Materials").mkdir(); (media / "Textures").mkdir()
    b = _textured_builder()
    path = gltf_export.export(b, str(media / "Models" / "scene.gltf"))
    plain = L.GltfScene(path)
    assert plain.desc.textureCount == 3 and plain.desc.textures[0].mipLevels > 1
    # 1. sibling: scene_tex0.dds next to scene_tex0.png (16 wide, 32 tall) with two mips of BC7 blocks
    sib = dds_dx10("BC7", 16, 32, rng.integers(0, 256, (4 * 8 + 2 * 4) * 16, dtype=np.uint8).tobytes(), mips=2)
    (media / "Models" / "scene_tex0.dds").write_bytes(sib)
    # 2. MSFT_texture_dds on the emissive texture (glTF texture 2)
    doc = json.loads(open(path).read())
    msft = dds_dx10("BC1", 8, 8, rng.integers(0, 256, 4 * 8, dtype=np.uint8).tobytes())
    (media / "Models" / "glow.dds").write_bytes(msft)
    doc["images"].append({"uri": "glow.dds"}); doc["textures"][2]["extensions"] = {"MSFT_texture_dds": {"source": len(doc["images"]) - 1}}
    open(path, "w").write(json.dumps(doc))
    g = L.GltfScene(path)
    assert g.desc.textureCount == 3
    t0 = g.desc.textures[0]; assert (t0.width, t0.height, t0.mipLevels, t0.format) == (16, 32, 2, S.FORMAT_RGBA8_SRGB)
    for m in range(2): np.testing.assert_array_equal(_texture_pixels(g.desc, 0, m), L.decode_dds(sib, m)[0])
    np.testing.assert_array_equal(_texture_pixels(g.desc, 1), _texture_pixels(plain.desc, 1))            # the normal map is still the PNG
    glow_slot = g.desc.materials[3].EmissiveTextureIndex & 0xFFFF
    np.testing.assert_array_equal(_texture_pixels(g.desc, glow_slot), L.decode_dds(msft)[0])
    idx = g.desc.materials[0].BaseOrDiffuseTextureIndex
    assert idx & 0xFFFF == 0 and (idx >> 16) & 0xFF == 2 and idx >> 24 == 9                             # log2(16*32) = 9, two mips (MaterialsBaker.cpp:499-501)
    g.close()
    # 3. material file: BaseTexture names a .png whose .dds sibling exists, NormalTexture a .png without one, the emissive file is missing (glTF texture kept)
    mat_name = doc["materials"][0]["name"]
    base_dds = dds_dx10("BC3", 8, 4, rng.integers(0, 256, 2 * 16, dtype=np.uint8).tobytes())
    (media / "Textures" / "albedo.dds").write_bytes(base_dds)
    nrm = rng.integers(0, 256, (4, 4, 4), dtype=np.uint8); nrm[..., 3] = 255
    (media / "Textures" / "bump.png").write_bytes(gltf_export.png_bytes(nrm))
    (media / "Materials" / ("%s.material.json" % mat_name)).write_text(json.dumps({
        "Roughness": 0.5, "BaseTexture": {"path": "Textures\\\\albedo.png", "sRGB": True}, "NormalTexture": {"path": "Textures/bump.png", "NormalMap": True},
        "EmissiveTexture": {"path": "Textures/missing.png", "sRGB": True}}))
    g = L.GltfScene(path, materials_dir=str(media / "Materials"))
    assert g.overridden_materials == 1
    m0 = g.desc.materials[0]
    assert m0.Flags & S.MATFLAG_UseBaseOrDiffuseTexture and m0.Flags & S.MATFLAG_UseNormalTexture and not (m0.Flags & S.MATFLAG_UseEmissiveTexture)
    bs, ns = m0.BaseOrDiffuseTextureIndex & 0xFFFF, m0.NormalTextureIndex & 0xFFFF
    tb = g.desc.textures[bs]; assert (tb.width, tb.height, tb.mipLevels, tb.format) == (8, 4, 1, S.FORMAT_RGBA8_SRGB)
    np.testing.assert_array_equal(_texture_pixels(g.desc, bs), L.decode_dds(base_dds)[0])
    tn = g.desc.textures[ns]; assert (tn.width, tn.height, tn.mipLevels, tn.format) == (4, 4, 3, S.FORMAT_RGBA8_UNORM)
    np.testing.assert_array_equal(_texture_pixels(g.desc, ns), nrm)
    g.close(); plain.close()


# ---- block-compressed textures kept compressed for the texture units (RTXPT_FORMAT_BC*) --------------------------------------------------------------------------------------
def _bc_scene(tmp_path, rng, fmt="BC7", size=(64, 64), mips=3):
    """The textured test scene with its base-colour PNG shadowed by a .dds sibling of random `fmt` blocks (sRGB slot)."""
    import sys, os
    sys.path.insert(0, os.path.dirname(__file__))
    import gltf_export
    from test_gltf_loader import _textured_builder
    d = tmp_path / ("m_" + fmt); d.mkdir()
    path = gltf_export.export(_textured_builder(), str(d / "scene.gltf"))
    w, h = size; payload = b""
    for m in range(mips):
        mw, mh = max(1, w >> m), max(1, h >> m)
        blocks = rng.integers(0, 256, (((mw + 3) // 4) * ((mh + 3) // 4), BLOCK_BYTES[fmt]), dtype=np.uint8)
        if fmt == "BC7": blocks[:, 0] = (blocks[:, 0] & 0x80) | 0x40            # mode 6: RGBA 7.7.7.7 + p-bits, one subset: every block is a smooth gradient (texture filtering stays well conditioned)
        payload += blocks.tobytes()
    file_bytes = dds_dx10(fmt, w, h, payload, mips=mips)
    (d / "scene_tex0.dds").write_bytes(file_bytes)
    return path, file_bytes


def test_loader_keeps_block_compression_when_asked(tmp_path):
    import ctypes as C
    from rtxpt_b200 import structs as S
    lib = L.load(); lib.rtxpt_b200_loader_keep_block_compression.argtypes = [C.c_int]; lib.rtxpt_b200_loader_keep_block_compression.restype = None
    rng = np.random.default_rng(21)
    for fmt, want in (("BC7", S.FORMAT_BC7_SRGB), ("BC1", S.FORMAT_BC1_SRGB), ("BC3", S.FORMAT_BC3_SRGB), ("BC2", S.FORMAT_BC2_SRGB)):
        path, file_bytes = _bc_scene(tmp_path, rng, fmt)
        try:
            lib.rtxpt_b200_loader_keep_block_compression(1); g = L.GltfScene(path)
        finally:
            lib.rtxpt_b200_loader_keep_block_compression(0)
        t = g.desc.textures[0]
        assert (t.width, t.height, t.mipLevels, t.format) == (64, 64, 3, want)                      # the base-colour slot is sRGB: the *_SRGB kind
        off = 148
        for m in range(3):
            n = ((max(1, 64 >> m) + 3) // 4) ** 2 * BLOCK_BYTES[fmt]
            assert C.string_at(t.mips[m], n) == file_bytes[off:off + n]; off += n                  # the raw blocks, untouched
        assert g.desc.textures[1].format == S.FORMAT_RGBA8_UNORM                                    # the PNG normal map is still RGBA8
        g.close()
        g = L.GltfScene(path); assert g.desc.textures[0].format == S.FORMAT_RGBA8_SRGB; g.close()  # default: expanded on the host
    # BC4 / BC5 and sizes that are not whole blocks always take the decoded path
    path, _ = _bc_scene(tmp_path, rng, "BC5")
    try:
        lib.rtxpt_b200_loader_keep_block_compression(1); g = L.GltfScene(path); assert g.desc.textures[0].format == S.FORMAT_RGBA8_SRGB; g.close()
    finally:
        lib.rtxpt_b200_loader_keep_block_compression(0)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["BC7", "BC3", "BC1"])
def test_block_compressed_textures_render_like_their_host_decode(tmp_path, fmt):
    """The same .dds once expanded to RGBA8 on the host, once kept compressed and decoded by the texture units: BC7 decodes exactly by specification, so the two frames agree to the
    filter's last bit; BC1 / BC3 colour interpolation may differ by one LSB between hardware and the reference decoder (the documented D3D tolerance)."""
    import ctypes as C
    from rtxpt_b200 import scene_builder as sb
    lib = L.load(); lib.rtxpt_b200_loader_keep_block_compression.argtypes = [C.c_int]; lib.rtxpt_b200_loader_keep_block_compression.restype = None
    path, _ = _bc_scene(tmp_path, np.random.default_rng(33), fmt, size=(128, 128), mips=5)
    frames = []
    for keep in (0, 1):
        try:
            lib.rtxpt_b200_loader_keep_block_compression(keep); g = L.GltfScene(path)
        finally:
            lib.rtxpt_b200_loader_keep_block_compression(0)
        cam = sb.bridge_camera(160, 120, pos=(0.0, 1.2, -3.5), direction=(0, -0.15, 1), up=(0, 1, 0), fov_y=0.9)
        consts = sb.make_constants(160, 120, cam, bounce_count=3, diffuse_bounce_count=3, env_enabled=False)
        c = L.Context(max_sub_samples_per_launch=4); c.upload_scene(g); c.set_constants(consts)
        c.path_trace(0, 8, True); c.synchronize(); frames.append(c.readback_accumulated()); c.close(); g.close()
    a, b = frames
    assert a[..., :3].mean() > 1e-3 and np.isfinite(b).all()
    rel = np.abs(a[..., :3] - b[..., :3]) / (np.abs(a[..., :3]) + 1e-2)
    if fmt == "BC7": assert np.percentile(rel, 99.9) < 2e-3 and abs(a.mean() - b.mean()) < 1e-4 * a.mean()
    else: assert np.percentile(rel, 99) < 5e-2 and abs(a.mean() - b.mean()) < 5e-3 * a.mean()          # the texture unit decodes BC1 / BC3 with its own rounding (one LSB of an sRGB-encoded colour is several percent of a dark linear value)
