"""ctypes binding of the product library librtxpt_b200.so (C ABI: include/rtxpt_b200.h).

There is no Python or CPU fallback: if the CUDA library is missing or no device is present, calls raise."""
import ctypes as C
import os
import subprocess
import numpy as np
from . import structs as S

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "_build", "librtxpt_b200.so")                  # default build (FMA, approximate div/sqrt)
LIB_PATH_STRICT = os.path.join(CSRC, "_build", "librtxpt_b200_strict.so")    # IEEE-exact arithmetic build, same sources and ABI (csrc/Makefile)


class RtxptError(RuntimeError):
    pass


def build(verbose=False):
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    r = subprocess.run(["make", "-C", CSRC, "-j4"], capture_output=not verbose, text=True)
    if r.returncode != 0:
        raise RtxptError("building librtxpt_b200.so failed:\n" + (r.stdout or "") + (r.stderr or ""))


_libs = {}

_SIGNATURES = {
    "rtxpt_b200_create": [C.POINTER(S.Config), C.POINTER(C.c_void_p)],
    "rtxpt_b200_destroy": [C.c_void_p],
    "rtxpt_b200_upload_scene": [C.c_void_p, C.POINTER(S.SceneDesc)],
    "rtxpt_b200_set_constants": [C.c_void_p, C.POINTER(S.PathTracerConstants)],
    "rtxpt_b200_path_trace": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p],
    "rtxpt_b200_reset_accumulation": [C.c_void_p],
    "rtxpt_b200_readback": [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t],
    "rtxpt_b200_device_ptr": [C.c_void_p, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)],
    "rtxpt_b200_synchronize": [C.c_void_p],
    "rtxpt_b200_render_frame": [C.c_void_p, C.POINTER(S.PathTracerConstants), C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t],
    "rtxpt_b200_get_stats": [C.c_void_p, C.POINTER(S.Stats)],
    "rtxpt_b200_tile_layout": [C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)],
    "rtxpt_b200_pack_owned": [C.c_void_p, C.c_void_p, C.c_void_p],
    "rtxpt_b200_unpack_all": [C.c_void_p, C.c_void_p, C.c_void_p],
    "rtxpt_b200_update_lights": [C.c_void_p, C.c_void_p, C.c_uint32],
    "rtxpt_b200_exchange_bytes": [C.c_void_p, C.POINTER(C.c_int), C.c_uint32, C.POINTER(C.c_size_t)],
    "rtxpt_b200_exchange_pack": [C.c_void_p, C.POINTER(C.c_int), C.c_uint32, C.c_void_p, C.c_void_p],
    "rtxpt_b200_exchange_unpack": [C.c_void_p, C.POINTER(C.c_int), C.c_uint32, C.c_void_p, C.c_void_p],
    "rtxpt_b200_trace_rays": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p],
    "rtxpt_b200_trace_rays_device": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_uint32, C.POINTER(C.c_float)],
    "rtxpt_b200_get_lights": [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)],
    "rtxpt_b200_set_view": [C.c_void_p, C.c_void_p],
    "rtxpt_b200_set_realtime": [C.c_void_p, C.POINTER(S.RealtimeConstants)],
    "rtxpt_b200_path_trace_realtime": [C.c_void_p, C.c_int, C.c_void_p],
    "rtxpt_b200_denoiser_prepare_inputs": [C.c_void_p, C.c_uint32, C.c_int, C.POINTER(S.DenoiserConstants), C.c_void_p],
    "rtxpt_b200_denoiser_final_merge": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p],
    "rtxpt_b200_skin_register": [C.c_void_p, C.POINTER(S.SkinDesc), C.POINTER(C.c_uint32)],
    "rtxpt_b200_skin_update": [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p],
    "rtxpt_b200_tone_map": [C.c_void_p, C.POINTER(S.ToneMappingParams), C.c_int, C.c_void_p],
    "rtxpt_b200_tone_map_average_luminance": [C.c_void_p, C.POINTER(C.c_float)],
    "rtxpt_b200_update_instance_transforms": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p],
    "rtxpt_b200_rebuild_bvh": [C.c_void_p, C.c_void_p],
    "rtxpt_b200_get_bvh_stats": [C.c_void_p, C.POINTER(S.BvhStats)],
    "rtxpt_b200_bake_env_map": [C.c_void_p, C.POINTER(S.EnvBakeDesc), C.c_void_p, C.c_size_t],
    "rtxpt_b200_neeat_update_begin": [C.c_void_p, C.c_void_p],
    "rtxpt_b200_neeat_update_end": [C.c_void_p, C.c_void_p],
    "rtxpt_b200_get_opacity_mask_stats": [C.c_void_p, C.POINTER(S.OpacityMaskStats)],
    "rtxpt_b200_host_bake_opacity_mask": [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p],
    "rtxpt_b200_neeat_reset": [C.c_void_p],
    "rtxpt_b200_neeat_readback": [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)],
    "rtxpt_b200_debug_scene_readback": [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)],
    "rtxpt_b200_neeat_debug_set_feedback": [C.c_void_p, C.c_void_p, C.c_void_p],
    "rtxpt_b200_denoise_spec_hit_t": [C.c_void_p, C.c_void_p],
    "rtxpt_b200_reblur_denoise": [C.c_void_p, C.c_uint32, C.POINTER(S.ReblurFrame), C.c_void_p],
    "rtxpt_b200_denoise_realtime": [C.c_void_p, C.POINTER(S.DenoiserConstants), C.POINTER(S.ReblurFrame), C.c_void_p],
    "rtxpt_b200_last_denoise_ms": [C.c_void_p, C.POINTER(C.c_float)],
    "rtxpt_b200_get_lights_ex": [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)],
    "rtxpt_b200_debug_bsdf": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p],
    "rtxpt_b200_debug_rng": [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p],
    "rtxpt_b200_debug_live_resources": [C.POINTER(C.c_uint64)],
}
_LOADER_SYMBOLS = ["rtxpt_b200_debug_decode_jpeg", "rtxpt_b200_debug_decode_jpeg_error", "rtxpt_b200_load_hdr_image", "rtxpt_b200_load_hdr_image_error", "rtxpt_b200_loader_keep_block_compression", "rtxpt_b200_load_dds_hdr", "rtxpt_b200_host_opacity_micro_index", "rtxpt_b200_camera_matrices", "rtxpt_b200_tone_map_pre_exposed_gray", "rtxpt_b200_debug_build_bvh", "rtxpt_b200_env_bake_mip_count", "rtxpt_b200_env_bake_floats", "rtxpt_b200_load_gltf", "rtxpt_b200_load_gltf_ex", "rtxpt_b200_load_scene_json", "rtxpt_b200_host_scene_info", "rtxpt_b200_load_gltf_error", "rtxpt_b200_host_scene_desc", "rtxpt_b200_host_scene_cameras",
                   "rtxpt_b200_host_scene_triangle_count", "rtxpt_b200_free_host_scene", "rtxpt_b200_bridge_camera", "rtxpt_b200_default_constants", "rtxpt_b200_debug_bvh_stats", "rtxpt_b200_parse_material_json", "rtxpt_b200_parse_material_json_error", "rtxpt_b200_debug_decode_dds", "rtxpt_b200_debug_decode_dds_error",
                    "rtxpt_b200_generic_ts_line_stride", "rtxpt_b200_generic_ts_plane_stride", "rtxpt_b200_generic_ts_address"]
EXPORTED_SYMBOLS = sorted(list(_SIGNATURES) + ["rtxpt_b200_last_error"] + _LOADER_SYMBOLS)


def load(strict=None):
    """Loads one of the two builds of the product; `strict=None` follows the RTXPT_STRICT environment variable (default: fast build)."""
    if strict is None:
        strict = os.environ.get("RTXPT_STRICT", "0") == "1"
    if strict not in _libs:
        path = LIB_PATH_STRICT if strict else LIB_PATH
        if os.environ.get("RTXPT_LIB_DIR"):        # tuning experiments: alternative builds of the same sources (make OUT=...)
            path = os.path.join(os.environ["RTXPT_LIB_DIR"], os.path.basename(path))
        if os.environ.get("RTXPT_LIB") and not strict:      # A/B measurement builds (csrc/Makefile `variant`)
            path = os.environ["RTXPT_LIB"]
        if not os.path.exists(path):
            raise RtxptError(f"{path} is missing: run rtxpt_b200.lib.build() / `make -C rtxpt_b200/csrc` (no fallback path exists)")
        L = C.CDLL(path)
        for name, args in _SIGNATURES.items():
            fn = getattr(L, name); fn.argtypes = args; fn.restype = C.c_int
        L.rtxpt_b200_last_error.restype = C.c_char_p
        L.rtxpt_b200_load_gltf.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]; L.rtxpt_b200_load_gltf.restype = C.c_int
        L.rtxpt_b200_load_gltf_error.restype = C.c_char_p
        L.rtxpt_b200_host_scene_desc.argtypes = [C.c_void_p]; L.rtxpt_b200_host_scene_desc.restype = C.POINTER(S.SceneDesc)
        L.rtxpt_b200_host_scene_cameras.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]; L.rtxpt_b200_host_scene_cameras.restype = C.c_int
        L.rtxpt_b200_host_scene_triangle_count.argtypes = [C.c_void_p]; L.rtxpt_b200_host_scene_triangle_count.restype = C.c_uint32
        L.rtxpt_b200_free_host_scene.argtypes = [C.c_void_p]; L.rtxpt_b200_free_host_scene.restype = None
        L.rtxpt_b200_bridge_camera.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, C.c_float,
                                               C.c_float, C.c_float, C.POINTER(C.c_float), C.POINTER(S.CameraData)]; L.rtxpt_b200_bridge_camera.restype = C.c_int
        L.rtxpt_b200_default_constants.argtypes = [C.POINTER(S.CameraData), C.c_int, C.POINTER(S.PathTracerConstants)]; L.rtxpt_b200_default_constants.restype = C.c_int
        _libs[strict] = L
    return _libs[strict]


def _check(rc, L=None):
    if rc != 0:
        raise RtxptError(f"rtxpt_b200 error {rc}: {(L or load()).rtxpt_b200_last_error().decode()}")


def bvh_stats(triangle_vertices, strict=None):
    """SAH statistics of the product's BVH over an (N, 3, 3) float32 triangle soup (host only)."""
    v = np.ascontiguousarray(triangle_vertices, np.float32).reshape(-1, 9)
    st = S.BvhStats(); L = load(strict)
    L.rtxpt_b200_debug_bvh_stats.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(S.BvhStats)]; L.rtxpt_b200_debug_bvh_stats.restype = C.c_int
    if L.rtxpt_b200_debug_bvh_stats(v.ctypes.data, len(v), C.byref(st)) != 0:
        raise RtxptError("bvh_stats failed")
    return st


def decode_dds(file_bytes, mip=0, strict=None):
    """DDS file bytes -> (HxWx4 uint8 RGBA of `mip`, mip count, srgb flag), host only."""
    L = load(strict); w, h, n, srgb = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    f = L.rtxpt_b200_debug_decode_dds; f.argtypes = [C.c_char_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]; f.restype = C.c_int
    L.rtxpt_b200_debug_decode_dds_error.restype = C.c_char_p
    if f(file_bytes, len(file_bytes), mip, C.byref(w), C.byref(h), C.byref(n), C.byref(srgb), None, 0) != 0:
        raise RtxptError("DDS: " + L.rtxpt_b200_debug_decode_dds_error().decode())
    out = np.empty((h.value, w.value, 4), np.uint8)
    if f(file_bytes, len(file_bytes), mip, C.byref(w), C.byref(h), C.byref(n), C.byref(srgb), out.ctypes.data, out.nbytes) != 0:
        raise RtxptError("DDS: " + L.rtxpt_b200_debug_decode_dds_error().decode())
    return out, n.value, bool(srgb.value)


def decode_jpeg(file_bytes, strict=None):
    """JPEG file bytes -> HxWx4 uint8 RGBA, host only (rtxpt_b200_debug_decode_jpeg: the glTF loader's decoder)."""
    L = load(strict); w, h = C.c_uint32(), C.c_uint32()
    f = L.rtxpt_b200_debug_decode_jpeg; f.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]; f.restype = C.c_int
    L.rtxpt_b200_debug_decode_jpeg_error.restype = C.c_char_p
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), None, 0) != 0: raise RtxptError("JPEG: " + L.rtxpt_b200_debug_decode_jpeg_error().decode())
    out = np.empty((h.value, w.value, 4), np.uint8)
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), out.ctypes.data, out.nbytes) != 0: raise RtxptError("JPEG: " + L.rtxpt_b200_debug_decode_jpeg_error().decode())
    return out


def load_dds_hdr(file_bytes, strict=None):
    """HDR DDS file bytes (BC6H UF16 / SF16, RGBA16F, RGBA32F; 2-D or cube) -> (faces x H x W x 4 float32 of mip 0, mip count), host only."""
    L = load(strict); w, h, faces, n = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    f = L.rtxpt_b200_load_dds_hdr; f.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]; f.restype = C.c_int
    L.rtxpt_b200_debug_decode_dds_error.restype = C.c_char_p
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), C.byref(faces), C.byref(n), None, 0) != 0:
        raise RtxptError("DDS: " + L.rtxpt_b200_debug_decode_dds_error().decode())
    out = np.empty((faces.value, h.value, w.value, 4), np.float32)
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), C.byref(faces), C.byref(n), out.ctypes.data, out.size) != 0:
        raise RtxptError("DDS: " + L.rtxpt_b200_debug_decode_dds_error().decode())
    return out, n.value


def load_hdr_image(file_bytes, strict=None):
    """OpenEXR / Radiance .hdr / HDR DDS file bytes -> H x W x 4 float32 (faces x H x W x 4 for a DDS cube), host only (rtxpt_b200_load_hdr_image)."""
    L = load(strict); w, h, faces = C.c_uint32(), C.c_uint32(), C.c_uint32()
    f = L.rtxpt_b200_load_hdr_image; f.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_void_p, C.c_uint64]; f.restype = C.c_int
    L.rtxpt_b200_load_hdr_image_error.restype = C.c_char_p
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), C.byref(faces), None, 0) != 0:
        raise RtxptError("image: " + L.rtxpt_b200_load_hdr_image_error().decode())
    out = np.empty((faces.value, h.value, w.value, 4), np.float32)
    if f(file_bytes, len(file_bytes), C.byref(w), C.byref(h), C.byref(faces), out.ctypes.data, out.size) != 0:
        raise RtxptError("image: " + L.rtxpt_b200_load_hdr_image_error().decode())
    return out[0] if faces.value == 1 else out


def parse_material_json(text, strict=None):
    """RTXPT .material.json text -> structs.MaterialJsonInfo (host only)."""
    L = load(strict); out = S.MaterialJsonInfo()
    L.rtxpt_b200_parse_material_json.argtypes = [C.c_char_p, C.POINTER(S.MaterialJsonInfo)]; L.rtxpt_b200_parse_material_json.restype = C.c_int
    L.rtxpt_b200_parse_material_json_error.restype = C.c_char_p
    if L.rtxpt_b200_parse_material_json(text.encode() if isinstance(text, str) else text, C.byref(out)) != 0:
        raise RtxptError("material JSON: " + L.rtxpt_b200_parse_material_json_error().decode())
    return out


class GltfScene:
    """A scene loaded by the library's host-side glTF loader (no GPU needed).  `.desc` is the RtxptSceneDesc to hand to Context.upload_scene
    (or to the oracle); `.cameras` lists the perspective cameras of the file."""
    def __init__(self, path, strict=None, materials_dir=None, scene_materials_dir=None, media_dir=None):
        self.L = load(strict)
        h = C.c_void_p(); n = C.c_uint32(0)
        self.L.rtxpt_b200_load_gltf_ex.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint32)]; self.L.rtxpt_b200_load_gltf_ex.restype = C.c_int
        enc = lambda p: None if p is None else os.fsencode(p)
        if str(path).endswith(".scene.json"):       # RTXPT scene file: models + graph + lights / cameras / settings; material files under <media>/Materials
            self.L.rtxpt_b200_load_scene_json.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]; self.L.rtxpt_b200_load_scene_json.restype = C.c_int
            rc = self.L.rtxpt_b200_load_scene_json(os.fsencode(path), enc(media_dir), C.byref(h))
        else:
            rc = self.L.rtxpt_b200_load_gltf_ex(os.fsencode(path), enc(materials_dir), enc(scene_materials_dir), C.byref(h), C.byref(n))
        self.overridden_materials = n.value
        if rc != 0:
            raise RtxptError("glTF load failed: " + self.L.rtxpt_b200_load_gltf_error().decode())
        self.h = h
        self.desc = self.L.rtxpt_b200_host_scene_desc(h).contents
        n = C.c_uint32(0); self.L.rtxpt_b200_host_scene_cameras(h, None, C.byref(n))
        cams = (S.GltfCamera * max(1, n.value))(); self.L.rtxpt_b200_host_scene_cameras(h, cams, C.byref(n))
        self.cameras = [cams[i] for i in range(n.value)]
        self.triangle_count = self.L.rtxpt_b200_host_scene_triangle_count(h)
        self.info = S.SceneFileInfo(); self.L.rtxpt_b200_host_scene_info.argtypes = [C.c_void_p, C.POINTER(S.SceneFileInfo)]; self.L.rtxpt_b200_host_scene_info(h, C.byref(self.info))
        self.material_count = self.desc.materialCount
        self.has_env = False

    def close(self):
        if self.h:
            self.L.rtxpt_b200_free_host_scene(self.h); self.h = None

    def __del__(self):
        try: self.close()
        except Exception: pass


def debug_build_bvh(triangle_vertices):
    """Host-only: the builder's BVH over a triangle soup (n x 9 float32).  Returns (nodes n x 20 u32, tris m x 12 u32 [v0 gid v1 flags v2 prim], levelStart)."""
    L = load(); v = np.ascontiguousarray(triangle_vertices, np.float32).reshape(-1, 9)
    f = L.rtxpt_b200_debug_build_bvh; f.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p] + [C.POINTER(C.c_uint32)] * 3; f.restype = C.c_int
    nn, nt, nl = C.c_uint32(), C.c_uint32(), C.c_uint32()
    assert f(v.ctypes.data, len(v), None, None, None, C.byref(nn), C.byref(nt), C.byref(nl)) == 0
    nodes = np.zeros((nn.value, 20), np.uint32); tris = np.zeros((nt.value, 12), np.uint32); levels = np.zeros(nl.value + 1, np.uint32)
    assert f(v.ctypes.data, len(v), nodes.ctypes.data, tris.ctypes.data, levels.ctypes.data, C.byref(nn), C.byref(nt), C.byref(nl)) == 0
    return nodes, tris, levels


def env_bake_arguments(cube_dim, source, source_type, scale_color, lights):
    """Shared by Context.bake_env_map and the test harnesses of the oracle / the host build: (source array or None, type, width, height, light table 8 floats each)."""
    src = None if source is None else np.ascontiguousarray(source, np.float32)
    if src is None: st, w, h = 0, 0, 0
    elif src.ndim == 4: st, w, h = 2, src.shape[1], src.shape[1]
    else: st, w, h = 1, src.shape[1], src.shape[0]
    if source_type is not None: st = source_type
    lt = np.zeros((len(lights), 8), np.float32)
    for i, (col, inten, direction, ang) in enumerate(lights): lt[i, :3] = col; lt[i, 3] = inten; lt[i, 4:7] = direction; lt[i, 7] = ang
    return src, st, w, h, lt


def split_env_mips(flat, cube_dim):
    out = []; off = 0; n = cube_dim
    while n > 0:
        cnt = 6 * n * n * 4; out.append(flat[off: off + cnt].reshape(6, n, n, 4)); off += cnt; n //= 2
    return out


def _bake_env_map(call, cube_dim, source, source_type, scale_color, lights):
    src, st, w, h, lt = env_bake_arguments(cube_dim, source, source_type, scale_color, lights)
    d = S.EnvBakeDesc(); d.cubeDim = cube_dim; d.sourceType = st; d.sourceWidth = w; d.sourceHeight = h; d.source = None if src is None else src.ctypes.data
    d.scaleColor[:] = list(scale_color); d.directionalLightCount = len(lt)
    for i in range(len(lt)): d.lights[i].colorIntensity[:] = lt[i, :4].tolist(); d.lights[i].direction[:] = lt[i, 4:7].tolist(); d.lights[i].angularSize = float(lt[i, 7])
    total = sum(6 * (cube_dim >> m) ** 2 * 4 for m in range(cube_dim.bit_length()))
    out = np.zeros(total, np.float32)
    call(d, out)
    return split_env_mips(out, cube_dim)


class Context:
    def __init__(self, max_sub_samples_per_launch=1, device=-1, tile_rank=0, tile_world=1, tile_size=64, flags=0, max_width=0, max_height=0, strict=None):
        L = self.L = load(strict)
        cfg = S.Config(device, max_width, max_height, max_sub_samples_per_launch, tile_rank, tile_world, tile_size, flags)
        self.h = C.c_void_p()
        _check(L.rtxpt_b200_create(C.byref(cfg), C.byref(self.h)))
        self.scene = None; self.consts = None

    def close(self):
        if self.h:
            self.L.rtxpt_b200_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def upload_scene(self, scene):
        self.scene = scene
        _check(self.L.rtxpt_b200_upload_scene(self.h, C.byref(scene.desc)), self.L)

    def set_constants(self, consts):
        self.consts = consts
        _check(self.L.rtxpt_b200_set_constants(self.h, C.byref(consts)), self.L)

    def path_trace(self, first_sub_sample, count, accumulate=True, stream=None):
        _check(self.L.rtxpt_b200_path_trace(self.h, first_sub_sample, count, int(accumulate), stream), self.L)

    def reset_accumulation(self):
        _check(self.L.rtxpt_b200_reset_accumulation(self.h), self.L)

    def synchronize(self):
        _check(self.L.rtxpt_b200_synchronize(self.h), self.L)

    def readback_accumulated(self, out=None):
        if out is None:
            out = np.empty((self.consts.imageHeight, self.consts.imageWidth, 4), np.float32)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_ACCUMULATED_F32, out.ctypes.data, out.nbytes), self.L)
        return out

    def set_view(self, world_to_clip):
        v = S.ViewConstants(); v.matWorldToClip[:] = [float(x) for x in np.asarray(world_to_clip, np.float32).reshape(16)]
        _check(self.L.rtxpt_b200_set_view(self.h, C.byref(v)), self.L)

    def readback_guides(self):
        """(depth f32 HxW, motion vectors f16 HxWx4, throughput u32 HxW packed R11G11B10) of the last sub-sample."""
        h, w = self.consts.imageHeight, self.consts.imageWidth
        depth = np.empty((h, w), np.float32); mv = np.empty((h, w, 4), np.float16); thp = np.empty((h, w), np.uint32)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_DEPTH_F32, depth.ctypes.data, depth.nbytes), self.L)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_MOTION_VECTORS_F16, mv.ctypes.data, mv.nbytes), self.L)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_THROUGHPUT_R11G11B10, thp.ctypes.data, thp.nbytes), self.L)
        return depth, mv, thp

    # ---- realtime mode (stable planes) ----
    def set_realtime(self, rt):
        self.realtime = rt
        _check(self.L.rtxpt_b200_set_realtime(self.h, C.byref(rt)), self.L)

    def path_trace_realtime(self, merge_no_denoiser=True, stream=None):
        """BUILD + rt.subSampleCount x FILL (+ the no-denoiser merge into the output colour)."""
        _check(self.L.rtxpt_b200_path_trace_realtime(self.h, 1 if merge_no_denoiser else 0, stream), self.L)

    def readback_realtime(self):
        """The realtime render targets as a dict of numpy arrays (same keys as the oracle's render_realtime)."""
        h, w = self.consts.imageHeight, self.consts.imageWidth
        plane_stride = self.L.rtxpt_b200_generic_ts_plane_stride(w, h)
        out = dict(planes=np.empty(3 * plane_stride, S.STABLE_PLANE_DTYPE), header=np.empty((4, h, w), np.uint32), stable_radiance=np.empty((h, w, 4), np.float16),
                   spec_hit_t=np.empty((h, w), np.float32))
        for key, buf in (("planes", S.BUFFER_STABLE_PLANES), ("header", S.BUFFER_STABLE_PLANES_HEADER), ("stable_radiance", S.BUFFER_STABLE_RADIANCE_F16), ("spec_hit_t", S.BUFFER_SPECULAR_HITT_F32)):
            _check(self.L.rtxpt_b200_readback(self.h, buf, out[key].ctypes.data, out[key].nbytes), self.L)
        out["depth"], out["motion"], out["throughput"] = self.readback_guides()
        out["merged"] = self.readback_output_color()[..., :3].astype(np.float32)
        return out

    # ---- RTXPT's side of the denoiser interface ----
    def denoiser_prepare_inputs(self, plane, init_with_stable_radiance, k, stream=None):
        _check(self.L.rtxpt_b200_denoiser_prepare_inputs(self.h, plane, 1 if init_with_stable_radiance else 0, C.byref(k), stream), self.L)

    def denoiser_final_merge(self, plane, d_diff=None, d_spec=None, stream=None, identity=True):
        """d_diff / d_spec: device pointers of RGBA16F images in NRD's output encoding.  Default (identity=True): the prepared inputs themselves (identity denoiser);
        identity=False passes NULL, NULL = the images reblur_denoise wrote."""
        if identity:
            if d_diff is None: d_diff = self.device_ptr(S.BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16)[0]
            if d_spec is None: d_spec = self.device_ptr(S.BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16)[0]
        _check(self.L.rtxpt_b200_denoiser_final_merge(self.h, plane, d_diff, d_spec, stream), self.L)

    def skin_register(self, instance, geometry, positions, joint_indices, joint_weights, normals=None, tangents=None):
        """Bind pose of one geometry (vertex order of its vertex buffer); returns the skin id for skin_update."""
        c = lambda a, t: None if a is None else np.ascontiguousarray(a, t)
        pos, ji, jw, nr, tg = c(positions, np.float32).reshape(-1, 3), c(joint_indices, np.uint16).reshape(-1, 4), c(joint_weights, np.float32).reshape(-1, 4), c(normals, np.uint32), c(tangents, np.uint32)
        d = S.SkinDesc(); d.instanceIndex = instance; d.geometryIndexInInstance = geometry; d.numVertices = len(pos)
        d.positions = pos.ctypes.data; d.jointIndices = ji.ctypes.data; d.jointWeights = jw.ctypes.data; d.normals = None if nr is None else nr.ctypes.data; d.tangents = None if tg is None else tg.ctypes.data
        sid = C.c_uint32(); _check(self.L.rtxpt_b200_skin_register(self.h, C.byref(d), C.byref(sid)), self.L)
        return int(sid.value)

    def skin_update(self, skin_id, joint_matrices, stream=None):
        m = np.ascontiguousarray(joint_matrices, np.float32).reshape(-1, 16)
        _check(self.L.rtxpt_b200_skin_update(self.h, skin_id, m.ctypes.data, len(m), stream), self.L)

    # (dtype, words per row) of rtxpt_b200_debug_scene_readback's buffers; 4 (the instance table) is returned as structs.InstanceData
    _SCENE_RAW = {0: (np.uint32, 20), 1: (np.uint32, 12), 2: (np.uint32, 24), 3: (np.float32, 9), 5: (np.uint32, 1), 6: (np.float32, 6)}

    def scene_raw(self, what):
        """Tests / debugging: the scene state on the device (0 BVH nodes, 1 leaf triangles, 2 shade records, 3 previous positions, 4 instances, 5 level starts, 6 exact node boxes);
        one row per node / triangle / record, level starts as a flat array."""
        n = C.c_size_t()
        _check(self.L.rtxpt_b200_debug_scene_readback(self.h, what, None, 0, C.byref(n)), self.L)
        if what == 4:
            out = (S.InstanceData * (n.value // C.sizeof(S.InstanceData)))()
            _check(self.L.rtxpt_b200_debug_scene_readback(self.h, what, out, n.value, C.byref(n)), self.L)
            return out
        dtype, row = self._SCENE_RAW[what]
        out = np.zeros(n.value // 4, dtype)
        _check(self.L.rtxpt_b200_debug_scene_readback(self.h, what, out.ctypes.data, out.nbytes, C.byref(n)), self.L)
        return out if row == 1 else out.reshape(-1, row)

    def tone_map(self, params, source=None, stream=None):
        """ToneMappingPass on the output colour (default) or the accumulation buffer; returns nothing - read the SRGBA8 result with readback_ldr()."""
        _check(self.L.rtxpt_b200_tone_map(self.h, C.byref(params), S.BUFFER_OUTPUT_COLOR_F16 if source is None else source, stream), self.L)

    def readback_ldr(self):
        out = np.empty((self.consts.imageHeight, self.consts.imageWidth, 4), np.uint8)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_LDR_COLOR_RGBA8, out.ctypes.data, out.nbytes), self.L)
        return out

    def tone_map_average_luminance(self):
        v = C.c_float(); _check(self.L.rtxpt_b200_tone_map_average_luminance(self.h, C.byref(v)), self.L); return float(v.value)

    def update_instance_transforms(self, transforms, stream=None):
        """transforms: instanceCount x 3 x 4 float32 (row-major): re-transforms the leaf triangles and refits the BVH on the stream."""
        t = np.ascontiguousarray(transforms, np.float32).reshape(-1, 12)
        _check(self.L.rtxpt_b200_update_instance_transforms(self.h, t.ctypes.data, len(t), stream), self.L)

    def rebuild_bvh(self, stream=None):
        """Rebuilds the BVH on the GPU over the leaf triangles as they are now (after update_instance_transforms / skin_update) and replaces the context's tree; returns with it in place."""
        _check(self.L.rtxpt_b200_rebuild_bvh(self.h, stream), self.L)

    def bvh_stats(self):
        """SAH statistics (structs.BvhStats) of the context's tree as it is now; buildSeconds: the last build (host at upload, or the device rebuild)."""
        st = S.BvhStats(); _check(self.L.rtxpt_b200_get_bvh_stats(self.h, C.byref(st)), self.L)
        return st

    def bake_env_map(self, cube_dim, source=None, source_type=None, scale_color=(1.0, 1.0, 1.0), lights=()):
        """EnvMapBaker on the GPU.  source: HxWx4 float32 equirectangular image or 6xNxNx4 cube (None = lights only); lights: (colour rgb, intensity W/sr, incoming direction,
        angular size rad) tuples.  Returns the MIP chain as a list of 6 x n x n x 4 float32 arrays (what SceneBuilder.set_env_cube / RtxptEnvCubeDesc take)."""
        return _bake_env_map(lambda d, out: _check(self.L.rtxpt_b200_bake_env_map(self.h, C.byref(d), out.ctypes.data, out.size), self.L), cube_dim, source, source_type, scale_color, lights)

    # ---- NEE-AT temporal feedback: per frame set_constants; neeat_update_begin; path_trace_realtime (runs update_end after its BUILD pass) ----
    def opacity_mask_stats(self):
        st = S.OpacityMaskStats(); _check(self.L.rtxpt_b200_get_opacity_mask_stats(self.h, C.byref(st)), self.L)
        return st

    def update_lights(self, lights):
        """lights: ctypes array of structs.LightDesc (or None): the scene's analytic lights of this frame (rtxpt_b200_update_lights)."""
        n = len(lights) if lights is not None else 0
        _check(self.L.rtxpt_b200_update_lights(self.h, lights if n else None, n), self.L)

    def neeat_update_begin(self, stream=None): _check(self.L.rtxpt_b200_neeat_update_begin(self.h, stream), self.L)

    def neeat_update_end(self, stream=None): _check(self.L.rtxpt_b200_neeat_update_end(self.h, stream), self.L)

    def neeat_reset(self): _check(self.L.rtxpt_b200_neeat_reset(self.h), self.L)

    def neeat_raw(self, what, dtype, count):
        """Same `what` codes as the oracle's oracle_neeat_get (0-1 feedback, 2-3 processed, 4-5 blended reservoirs, 6 tile lists, 7 proxy counters, 8 control, 11 proxy table)."""
        a = np.zeros(count, dtype); n = C.c_size_t()
        _check(self.L.rtxpt_b200_neeat_readback(self.h, what, a.ctypes.data, a.nbytes, C.byref(n)), self.L)
        return a[: n.value // a.itemsize]

    def neeat_set_feedback(self, weight, candidate):
        w = np.ascontiguousarray(weight, np.float32); c = np.ascontiguousarray(candidate, np.uint32)
        _check(self.L.rtxpt_b200_neeat_debug_set_feedback(self.h, w.ctypes.data, c.ctypes.data), self.L)

    def denoise_spec_hit_t(self, stream=None):
        _check(self.L.rtxpt_b200_denoise_spec_hit_t(self.h, stream), self.L)

    # ---- ReBLUR ----
    def reblur_denoise(self, plane, frame, stream=None):
        _check(self.L.rtxpt_b200_reblur_denoise(self.h, plane, C.byref(frame), stream), self.L)

    def denoise_realtime(self, k, frame, stream=None):
        """Sample::Denoise: for plane = active-1..0 { prepare inputs; ReBLUR; final merge } into the output colour."""
        _check(self.L.rtxpt_b200_denoise_realtime(self.h, C.byref(k), C.byref(frame), stream), self.L)

    def last_denoise_ms(self):
        ms = C.c_float()
        _check(self.L.rtxpt_b200_last_denoise_ms(self.h, C.byref(ms)), self.L)
        return float(ms.value)

    def readback_reblur(self):
        h, w = self.consts.imageHeight, self.consts.imageWidth
        out = dict(diff=np.empty((h, w, 4), np.float16), spec=np.empty((h, w, 4), np.float16), frames=np.empty((h, w, 2), np.uint8))
        for key, buf in (("diff", S.BUFFER_DENOISED_DIFF_RADIANCE_HITDIST_F16), ("spec", S.BUFFER_DENOISED_SPEC_RADIANCE_HITDIST_F16), ("frames", S.BUFFER_REBLUR_ACCUMULATED_FRAMES_RG8)):
            _check(self.L.rtxpt_b200_readback(self.h, buf, out[key].ctypes.data, out[key].nbytes), self.L)
        out["frames"] = out["frames"].astype(np.float32) / 255.0 * 63.0
        return out

    def readback_denoiser_inputs(self):
        h, w = self.consts.imageHeight, self.consts.imageWidth
        out = dict(view_z=np.empty((h, w), np.float32), motion=np.empty((h, w, 4), np.float16), normal_roughness=np.empty((h, w), np.uint32), diff=np.empty((h, w, 4), np.float16),
                   spec=np.empty((h, w, 4), np.float16), disocclusion_mix=np.empty((h, w), np.uint8), history_clamp_relax=np.empty((h, w), np.uint8))
        for key, buf in (("view_z", S.BUFFER_DENOISER_VIEWSPACE_Z_F32), ("motion", S.BUFFER_DENOISER_MOTION_VECTORS_F16), ("normal_roughness", S.BUFFER_DENOISER_NORMAL_ROUGHNESS_R10G10B10A2),
                         ("diff", S.BUFFER_DENOISER_DIFF_RADIANCE_HITDIST_F16), ("spec", S.BUFFER_DENOISER_SPEC_RADIANCE_HITDIST_F16), ("disocclusion_mix", S.BUFFER_DENOISER_DISOCCLUSION_MIX_R8),
                         ("history_clamp_relax", S.BUFFER_COMBINED_HISTORY_CLAMP_RELAX_R8)):
            _check(self.L.rtxpt_b200_readback(self.h, buf, out[key].ctypes.data, out[key].nbytes), self.L)
        return out

    def readback_output_color(self):
        out = np.empty((self.consts.imageHeight, self.consts.imageWidth, 4), np.float16)
        _check(self.L.rtxpt_b200_readback(self.h, S.BUFFER_OUTPUT_COLOR_F16, out.ctypes.data, out.nbytes), self.L)
        return out

    def device_ptr(self, buffer):
        p, n = C.c_void_p(), C.c_size_t()
        _check(self.L.rtxpt_b200_device_ptr(self.h, buffer, C.byref(p), C.byref(n)), self.L)
        return p.value, n.value

    def render_frame(self, consts, first_sub_sample, count, out=None):
        self.consts = consts
        if out is None:
            out = np.empty((consts.imageHeight, consts.imageWidth, 4), np.float32)
        _check(self.L.rtxpt_b200_render_frame(self.h, C.byref(consts), first_sub_sample, count, out.ctypes.data, out.nbytes), self.L)
        return out

    def stats(self):
        st = S.Stats()
        _check(self.L.rtxpt_b200_get_stats(self.h, C.byref(st)), self.L)
        return st

    def tile_layout(self):
        a, b = C.c_uint32(), C.c_uint32()
        _check(self.L.rtxpt_b200_tile_layout(self.h, C.byref(a), C.byref(b)), self.L)
        return a.value, b.value

    def pack_owned(self, d_dst, stream=None):
        _check(self.L.rtxpt_b200_pack_owned(self.h, d_dst, stream), self.L)

    def unpack_all(self, d_src_all, stream=None):
        _check(self.L.rtxpt_b200_unpack_all(self.h, d_src_all, stream), self.L)

    # ---- multi-GPU exchange of the realtime frame's per-pixel images (rtxpt_b200_exchange_*) ----
    def _ids(self, buffers):
        return (C.c_int * len(buffers))(*buffers), len(buffers)

    def exchange_bytes(self, buffers):
        ids, n = self._ids(buffers); out = C.c_size_t()
        _check(self.L.rtxpt_b200_exchange_bytes(self.h, ids, n, C.byref(out)), self.L)
        return out.value

    def exchange_pack(self, buffers, d_dst, stream=None):
        ids, n = self._ids(buffers); _check(self.L.rtxpt_b200_exchange_pack(self.h, ids, n, d_dst, stream), self.L)

    def exchange_unpack(self, buffers, d_src_all, stream=None):
        ids, n = self._ids(buffers); _check(self.L.rtxpt_b200_exchange_unpack(self.h, ids, n, d_src_all, stream), self.L)

    def trace_rays(self, rays, any_hit=False):
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 8)
        hits = np.zeros(len(rays), dtype=[("t", "f4"), ("u", "f4"), ("v", "f4"), ("inst", "u4"), ("geom", "u4"), ("prim", "u4")])
        _check(self.L.rtxpt_b200_trace_rays(self.h, rays.ctypes.data, len(rays), int(any_hit), hits.ctypes.data), self.L)
        return hits

    def trace_rays_device(self, d_rays, count, d_hits, any_hit=False, repeat=1):
        ms = C.c_float()
        _check(self.L.rtxpt_b200_trace_rays_device(self.h, d_rays, count, int(any_hit), d_hits, repeat, C.byref(ms)), self.L)
        return ms.value

    def lights(self):
        n, m = C.c_uint32(0), C.c_uint32(0)
        _check(self.L.rtxpt_b200_get_lights(self.h, None, C.byref(n), None, None, C.byref(m)), self.L)
        infos = np.zeros((n.value, 8), np.uint32); counters = np.zeros(n.value, np.uint32); proxies = np.zeros(max(m.value, 1), np.uint32)
        _check(self.L.rtxpt_b200_get_lights(self.h, infos.ctypes.data, C.byref(n), counters.ctypes.data, proxies.ctypes.data, C.byref(m)), self.L)
        return infos, counters, proxies[:m.value]

    def lights_ex(self):
        n = C.c_uint32(0)
        _check(self.L.rtxpt_b200_get_lights_ex(self.h, None, C.byref(n)), self.L)
        ex = np.zeros((n.value, 4), np.uint32)
        if n.value:
            _check(self.L.rtxpt_b200_get_lights_ex(self.h, ex.ctypes.data, C.byref(n)), self.L)
        return ex

    def debug_bsdf(self, records):
        records = np.ascontiguousarray(records, np.float32).reshape(-1, 36)
        out = np.zeros((len(records), 16), np.float32)
        _check(self.L.rtxpt_b200_debug_bsdf(self.h, records.ctypes.data, len(records), out.ctypes.data), self.L)
        return out

    def debug_rng(self, tuples):
        tuples = np.ascontiguousarray(tuples, np.uint32).reshape(-1, 4)
        out = np.zeros((len(tuples), 8), np.uint32)
        _check(self.L.rtxpt_b200_debug_rng(self.h, tuples.ctypes.data, len(tuples), out.ctypes.data), self.L)
        return out
