"""Builds the GPU-table view of a scene (the data contract of the PathTrace dispatch, Rtxpt/Sample.cpp:2315-2427) from numpy
meshes.  It plays the role Donut's Scene::CreateMeshBuffers / MaterialsBaker::Update play in the reference
(External/Donut/src/engine/Scene.cpp:821-1000, Rtxpt/Materials/MaterialsBaker.cpp:516-591, :960-1017): SoA vertex buffers with
snorm8 normals/tangents (External/Donut/src/core/math/vector.cpp:84-103), GeometryData / InstanceData / SubInstanceData /
PTMaterialData tables.  Used by the tests, bench.py and the synthetic stand-in scenes; the C++ glTF host path produces the same
tables."""
import ctypes as C
import math
import numpy as np
from . import structs as S


def pack_snorm8_vec3(v):
    """vectorToSnorm8<3>: truncating int(v * 127/|v|), External/Donut/src/core/math/vector.cpp:84-92."""
    v = np.asarray(v, np.float32)
    ln = np.sqrt((v * v).sum(-1, keepdims=True)).astype(np.float32)
    scale = np.float32(127.0) / np.maximum(ln, np.float32(1e-30))
    q = np.trunc(v * scale).astype(np.int32) & 0xff
    return (q[..., 0] | (q[..., 1] << 8) | (q[..., 2] << 16)).astype(np.uint32)


def pack_snorm8_vec4(v):
    v = np.asarray(v, np.float32)
    ln = np.sqrt((v[..., :3] * v[..., :3]).sum(-1, keepdims=True)).astype(np.float32)
    scale = np.float32(127.0) / np.maximum(ln, np.float32(1e-30))
    q = np.trunc(v * scale).astype(np.int32) & 0xff
    return (q[..., 0] | (q[..., 1] << 8) | (q[..., 2] << 16) | (q[..., 3] << 24)).astype(np.uint32)


def compute_tangents(positions, uvs, normals, indices):
    """Per-vertex tangents the way GltfImporter builds them when the asset has none (GltfImporter.cpp:1331-1421)."""
    p = positions.astype(np.float32); t = uvs.astype(np.float32); tri = indices.reshape(-1, 3)
    p0, p1, p2 = p[tri[:, 0]], p[tri[:, 1]], p[tri[:, 2]]
    t0, t1, t2 = t[tri[:, 0]], t[tri[:, 1]], t[tri[:, 2]]
    dPds, dPdt = p1 - p0, p2 - p0
    dTds, dTdt = t1 - t0, t2 - t0
    det = dTds[:, 0] * dTdt[:, 1] - dTds[:, 1] * dTdt[:, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        r = (1.0 / det)[:, None]
        tangent = r * (dPds * dTdt[:, 1:2] - dPdt * dTds[:, 1:2])
        bitangent = r * (dPdt * dTds[:, 0:1] - dPds * dTdt[:, 0:1])
    tl = np.linalg.norm(tangent, axis=1); bl = np.linalg.norm(bitangent, axis=1)
    ok = np.isfinite(tl) & np.isfinite(bl) & (tl > 0) & (bl > 0)
    tangent = np.where(ok[:, None], tangent / np.where(ok, tl, 1)[:, None], 0)
    bitangent = np.where(ok[:, None], bitangent / np.where(ok, bl, 1)[:, None], 0)
    T = np.zeros_like(p); B = np.zeros_like(p)
    for k in range(3):
        np.add.at(T, tri[:, k], tangent); np.add.at(B, tri[:, k], bitangent)
    tl = np.linalg.norm(T, axis=1); bl = np.linalg.norm(B, axis=1)
    ok = (tl > 0) & (bl > 0)
    Tn = np.where(ok[:, None], T / np.where(ok, tl, 1)[:, None], 0)
    Bn = np.where(ok[:, None], B / np.where(ok, bl, 1)[:, None], 0)
    sign = np.where(ok, np.where((np.cross(normals, Tn) * Bn).sum(1) > 0, -1.0, 1.0), 0.0)
    return np.concatenate([Tn, sign[:, None]], axis=1).astype(np.float32)


def make_mips_u8(img):
    """Box-filtered mip chain of an HxWx4 uint8 image down to 1x1 (the authored mip chains of the reference's DDS assets)."""
    mips = [np.ascontiguousarray(img, dtype=np.uint8)]
    cur = img.astype(np.float32)
    while cur.shape[0] > 1 or cur.shape[1] > 1:
        h, w = cur.shape[0], cur.shape[1]
        nh, nw = max(1, h // 2), max(1, w // 2)
        c = cur[: nh * 2 if h > 1 else 1, : nw * 2 if w > 1 else 1]
        if h > 1 and w > 1:
            c = (c[0::2, 0::2] + c[1::2, 0::2] + c[0::2, 1::2] + c[1::2, 1::2]) * 0.25
        elif h > 1:
            c = (c[0::2] + c[1::2]) * 0.5
        else:
            c = (c[:, 0::2] + c[:, 1::2]) * 0.5
        cur = c
        mips.append(np.ascontiguousarray(np.clip(np.rint(cur), 0, 255).astype(np.uint8)))
    return mips


def make_cube_mips(faces):
    """faces: 6xNxNx4 float32 -> list (per mip) of 6xnxnx4 arrays, 2x2 box filter."""
    out = [np.ascontiguousarray(faces, dtype=np.float32)]
    cur = out[0]
    while cur.shape[1] > 1:
        cur = np.ascontiguousarray((cur[:, 0::2, 0::2] + cur[:, 1::2, 0::2] + cur[:, 0::2, 1::2] + cur[:, 1::2, 1::2]) * np.float32(0.25))
        out.append(cur)
    return out


def identity34():
    return np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float32)


def translate_scale(t, s=(1, 1, 1)):
    m = identity34(); m[0, 0], m[1, 1], m[2, 2] = s; m[:, 3] = t
    return m


class Material:
    """Subset of PTMaterial (Rtxpt/Materials/MaterialsBaker.h) that reaches PTMaterialData through FillData."""
    def __init__(self, base_color=(1, 1, 1), roughness=1.0, metalness=0.0, emissive=(0, 0, 0), emissive_intensity=1.0,
                 transmission=0.0, diffuse_transmission=0.0, ior=1.5, thin_surface=False, opacity=1.0, alpha_test=False, alpha_cutoff=0.5,
                 base_texture=None, orm_texture=None, normal_texture=None, emissive_texture=None, nested_priority=0,
                 volume_color=(1, 1, 1), volume_distance=3.4e38, shadow_nol_fadeout=0.0, exclude_from_nee=False, normal_scale=1.0,
                 metalness_in_red=False, analytic_light_proxy=False, psd_exclude=True, psd_dominant_delta_lobe=-1, psd_block_mvs_at_surface=0):
        self.__dict__.update(locals()); del self.__dict__["self"]

    @property
    def enable_transmission(self):
        return self.transmission > 0 or self.diffuse_transmission > 0


class SceneBuilder:
    def __init__(self):
        self.textures = []      # (mips list, format)
        self.materials = []
        self.meshes = []        # list of geometries: dict(positions, uvs, normals, tangents, indices, material)
        self.instances = []     # (mesh index, 3x4 transform)
        self.env_faces = None
        self.lights = []        # analytic lights: dicts with the RtxptLightDesc fields

    def add_point_light(self, position, color, intensity, radius):
        """Donut PointLight + RTXPT radius extension; radius > 0 makes it a sphere light (LightsBaker.cpp:528-551)."""
        self.lights.append(dict(type=S.LIGHT_POINT, position=position, direction=(0, 0, -1), color=color, intensity=intensity, radius=radius, inner=0.0, outer=0.0))

    def add_spot_light(self, position, direction, color, intensity, radius, inner_angle, outer_angle):
        """Donut SpotLight (angles in degrees); a sphere light with cone shaping (LightsBaker.cpp:463-500)."""
        self.lights.append(dict(type=S.LIGHT_SPOT, position=position, direction=direction, color=color, intensity=intensity, radius=radius, inner=inner_angle, outer=outer_angle))

    def add_texture(self, img_u8, srgb):
        self.textures.append((make_mips_u8(img_u8), S.FORMAT_RGBA8_SRGB if srgb else S.FORMAT_RGBA8_UNORM))
        return len(self.textures) - 1

    def add_material(self, mat):
        self.materials.append(mat)
        return len(self.materials) - 1

    def add_mesh(self, geometries):
        """geometries: list of dicts with positions (Nx3), indices (Mx3), normals (Nx3), optional uvs (Nx2), tangents (Nx4), material"""
        self.meshes.append(geometries)
        return len(self.meshes) - 1

    def add_instance(self, mesh, transform=None, proxy_light=None):
        """proxy_light: index (into the analytic lights added so far) of the light this instance's proxy-flagged geometry stands in for."""
        self.instances.append((mesh, identity34() if transform is None else np.asarray(transform, np.float32).reshape(3, 4)))
        self.instance_proxy_light = getattr(self, "instance_proxy_light", {}); self.instance_proxy_light[len(self.instances) - 1] = proxy_light

    def set_env_cube(self, faces):
        self.env_faces = np.asarray(faces, np.float32)

    def _tex_info(self, idx):
        mips, _ = self.textures[idx]
        h, w = mips[0].shape[0], mips[0].shape[1]
        base_lod = int(math.log2(float(w * h)) + 0.5)           # MaterialsBaker.cpp:499-501
        return (base_lod << 24) | (len(mips) << 16) | idx

    def build(self):
        return Scene(self)


def make_light_array(lights):
    """List of light dicts (SceneBuilder.add_point_light / add_spot_light fields) -> ctypes array of RtxptLightDesc: the `lights` of a scene, or of rtxpt_b200_update_lights."""
    arr = (S.LightDesc * len(lights))()
    for l, L in zip(arr, lights):
        l.type = L["type"]; l.position[:] = L["position"]; l.direction[:] = L["direction"]; l.color[:] = L["color"]
        l.intensity, l.radius, l.innerAngle, l.outerAngle = L["intensity"], L["radius"], L["inner"], L["outer"]
    return arr


def point_light(position, color, intensity, radius):
    return dict(type=S.LIGHT_POINT, position=position, direction=(0, 0, -1), color=color, intensity=intensity, radius=radius, inner=0.0, outer=0.0)


class Scene:
    """Owns the numpy storage behind an RtxptSceneDesc (`.desc`)."""
    def __init__(self, b):
        self._keep = []
        # textures
        self.tex_descs = (S.TextureDesc * max(1, len(b.textures)))()
        for i, (mips, fmt) in enumerate(b.textures):
            d = self.tex_descs[i]
            d.width, d.height, d.mipLevels, d.format = mips[0].shape[1], mips[0].shape[0], len(mips), fmt
            for m, arr in enumerate(mips):
                self._keep.append(arr); d.mips[m] = arr.ctypes.data
        # materials (PTMaterial::FillData, MaterialsBaker.cpp:516-591)
        self.materials = (S.MaterialData * max(1, len(b.materials)))()
        for i, m in enumerate(b.materials):
            d = self.materials[i]
            flags = 0
            def tex(idx, bit):
                nonlocal flags
                if idx is None:
                    return 0xFFFFFFFF
                flags |= bit
                return b._tex_info(idx)
            d.BaseOrDiffuseTextureIndex = tex(m.base_texture, S.MATFLAG_UseBaseOrDiffuseTexture)
            d.MetalRoughOrSpecularTextureIndex = tex(m.orm_texture, S.MATFLAG_UseMetalRoughOrSpecularTexture)
            d.EmissiveTextureIndex = tex(m.emissive_texture, S.MATFLAG_UseEmissiveTexture)
            d.NormalTextureIndex = tex(m.normal_texture, S.MATFLAG_UseNormalTexture)
            d.TransmissionTextureIndex = 0xFFFFFFFF
            d.OcclusionTextureIndex = 0xFFFFFFFF
            if m.metalness_in_red:
                flags |= S.MATFLAG_MetalnessInRedChannel
            if m.analytic_light_proxy:
                flags |= S.MATFLAG_EnableAsAnalyticLightProxy
            if m.thin_surface or not m.enable_transmission:      # MaterialsBaker.cpp:543-544
                flags |= S.MATFLAG_ThinSurface
            flags |= (min(int(m.nested_priority), 14) & 0xF) << S.MATFLAG_NestedPriorityShift
            # path-space decomposition controls of realtime mode (MaterialsBaker.h:173-177 defaults: excluded, no dominant lobe, motion vectors not blocked;
            # FillData MaterialsBaker.cpp:546-553, :586)
            if m.psd_exclude:
                flags |= S.MATFLAG_PSDExclude
            flags |= (int(m.psd_block_mvs_at_surface) % 2) << 13 | (int(m.psd_block_mvs_at_surface) // 2) << 14
            flags |= min(max(int(m.psd_dominant_delta_lobe) + 1, 0), 7) << 24
            d.Flags = flags
            d.BaseOrDiffuseColor[:] = m.base_color
            d.SpecularColor[:] = (0, 0, 0)
            d.EmissiveColor[:] = [np.float32(c) * np.float32(m.emissive_intensity) for c in m.emissive]
            d.Roughness, d.Metalness, d.NormalTextureScale = m.roughness, m.metalness, m.normal_scale
            d.TransmissionFactor = m.transmission if m.enable_transmission else 0.0
            d.DiffuseTransmissionFactor = m.diffuse_transmission if m.enable_transmission else 0.0
            d.Opacity, d.AlphaCutoff, d.IoR = m.opacity, m.alpha_cutoff, m.ior
            d.VolumeAttenuationColor[:] = m.volume_color
            d.VolumeAttenuationDistance = min(m.volume_distance, 3.4e38)
            d.ShadowNoLFadeout = min(max(m.shadow_nol_fadeout, 0.0), 0.25)
            d._padding0 = 42; d._padding1 = 42.0
        # meshes -> buffers + geometries
        n_geo = sum(len(g) for g in b.meshes)
        self.geometries = (S.GeometryData * max(1, n_geo))()
        self.buffers = (S.BufferDesc * max(1, 2 * len(b.meshes)))()
        mesh_first_geo = []
        gi = 0
        self.triangle_count = 0
        for mi, geos in enumerate(b.meshes):
            mesh_first_geo.append(gi)
            nv = sum(len(g["positions"]) for g in geos)
            idx_blob = np.concatenate([np.asarray(g["indices"], np.uint32).reshape(-1) for g in geos])
            pos = np.concatenate([np.asarray(g["positions"], np.float32) for g in geos]).astype(np.float32)
            has_uv = all(g.get("uvs") is not None for g in geos)
            uvs = np.concatenate([np.asarray(g["uvs"], np.float32) for g in geos]) if has_uv else np.zeros((nv, 2), np.float32)
            nrm = np.concatenate([np.asarray(g["normals"], np.float32) for g in geos])
            tans = []
            for g in geos:
                t = g.get("tangents")
                if t is None:
                    t = compute_tangents(np.asarray(g["positions"], np.float32), np.asarray(g["uvs"], np.float32), np.asarray(g["normals"], np.float32),
                                         np.asarray(g["indices"], np.uint32)) if g.get("uvs") is not None else np.zeros((len(g["positions"]), 4), np.float32)
                tans.append(np.asarray(t, np.float32))
            tan = np.concatenate(tans)
            off_pos, off_uv = 0, nv * 12
            off_nrm, off_tan = off_uv + nv * 8, off_uv + nv * 8 + nv * 4
            # optional previous-position stream (Donut keeps one for skinned meshes: GeometryData.prevPositionOffset): geometries that give "prev_positions"
            has_prev = any(g.get("prev_positions") is not None for g in geos); off_prev = off_tan + nv * 4
            vblob = np.zeros(off_prev + (nv * 12 if has_prev else 0), np.uint8)
            if has_prev:
                prev = np.concatenate([np.asarray(g["prev_positions"] if g.get("prev_positions") is not None else g["positions"], np.float32) for g in geos]).astype(np.float32)
                vblob[off_prev:] = prev.reshape(-1).view(np.uint8)
            vblob[off_pos:off_uv] = pos.reshape(-1).view(np.uint8)
            vblob[off_uv:off_nrm] = np.ascontiguousarray(uvs, np.float32).reshape(-1).view(np.uint8)
            vblob[off_nrm:off_tan] = pack_snorm8_vec3(nrm).view(np.uint8)
            vblob[off_tan:off_prev] = pack_snorm8_vec4(tan).view(np.uint8)
            idx_blob = np.ascontiguousarray(idx_blob); self._keep += [idx_blob, vblob]
            self.buffers[2 * mi].data, self.buffers[2 * mi].sizeBytes = idx_blob.ctypes.data, idx_blob.nbytes
            self.buffers[2 * mi + 1].data, self.buffers[2 * mi + 1].sizeBytes = vblob.ctypes.data, vblob.nbytes
            v0 = 0; i0 = 0
            for g in geos:
                d = self.geometries[gi]
                n_i = np.asarray(g["indices"]).size; n_v = len(g["positions"])
                d.numIndices, d.numVertices = n_i, n_v
                d.indexBufferIndex, d.indexOffset = 2 * mi, i0 * 4
                d.vertexBufferIndex = 2 * mi + 1
                d.positionOffset = off_pos + v0 * 12
                d.prevPositionOffset = (off_prev + v0 * 12) if g.get("prev_positions") is not None else 0xFFFFFFFF
                d.texCoord1Offset = (off_uv + v0 * 8) if has_uv else 0xFFFFFFFF
                d.texCoord2Offset = 0xFFFFFFFF
                d.normalOffset = off_nrm + v0 * 4
                d.tangentOffset = off_tan + v0 * 4
                d.curveRadiusOffset = 0xFFFFFFFF
                d.materialIndex = g["material"]
                v0 += n_v; i0 += n_i; gi += 1
        # instances + sub-instances (UpdateSubInstanceData, MaterialsBaker.cpp:960-1017)
        n_sub = sum(len(b.meshes[m]) for m, _ in b.instances)
        self.instances = (S.InstanceData * max(1, len(b.instances)))()
        self.sub_instances = (S.SubInstanceData * max(1, n_sub))()
        si = 0
        for ii, (mi, xf) in enumerate(b.instances):
            d = self.instances[ii]
            d.flags, d.firstGeometryInstanceIndex, d.firstGeometryIndex, d.numGeometries = 0, si, mesh_first_geo[mi], len(b.meshes[mi])
            pxf = getattr(b, "prev_transforms", {}).get(ii, xf)            # last frame's matrix (Donut's InstanceData.prevTransform); default: the instance did not move
            d.transform[:] = xf.reshape(-1).tolist(); d.prevTransform[:] = np.asarray(pxf, np.float32).reshape(-1).tolist()
            for k, g in enumerate(b.meshes[mi]):
                s = self.sub_instances[si]
                mat = b.materials[g["material"]]
                geo = self.geometries[mesh_first_geo[mi] + k]
                alpha = mat.alpha_test and mat.base_texture is not None
                fl = 0; cutoff = 0.0
                if alpha:
                    fl |= S.SUBINST_FLAG_ALPHA_TESTED | (mat.base_texture & 0xFFFF); cutoff = mat.alpha_cutoff
                fl |= int(min(max(cutoff, 0.0), 1.0) * 255.0 + 0.5) << 24
                if mat.exclude_from_nee:
                    fl |= S.SUBINST_FLAG_EXCLUDE_FROM_NEE
                s.FlagsAndAlphaInfo = fl
                s.GlobalGeometryIndex_PTMaterialDataIndex = ((mesh_first_geo[mi] + k) << 16) | g["material"]
                s.EmissiveLightMappingOffset = 0xFFFFFFFF
                pl = getattr(b, "instance_proxy_light", {}).get(ii)
                s.AnalyticProxyLightIndex = 0xFFFFFFFF if (pl is None or not mat.analytic_light_proxy) else pl
                s.IndexBufferIndex_VertexBufferIndex = (geo.indexBufferIndex << 16) | geo.vertexBufferIndex
                s.IndexOffset, s.TexCoord1Offset = geo.indexOffset, geo.texCoord1Offset
                self.triangle_count += geo.numIndices // 3
                si += 1
        d = S.SceneDesc()
        d.instances, d.instanceCount = self.instances, len(b.instances)
        d.geometries, d.geometryCount = self.geometries, n_geo
        d.subInstances, d.subInstanceCount = self.sub_instances, n_sub
        d.materials, d.materialCount = self.materials, len(b.materials)
        d.buffers, d.bufferCount = self.buffers, 2 * len(b.meshes)
        d.textures, d.textureCount = self.tex_descs, len(b.textures)
        if b.env_faces is not None:
            mips = make_cube_mips(b.env_faces)
            d.envCube.faceSize, d.envCube.mipLevels = b.env_faces.shape[1], len(mips)
            for m, arr in enumerate(mips):
                self._keep.append(arr)
                for f in range(6):
                    d.envCube.faces[f][m] = arr[f].ctypes.data
        self.lights = make_light_array(b.lights) if b.lights else (S.LightDesc * 1)()
        d.lights, d.lightCount = self.lights, len(b.lights)
        self.desc = d
        self.material_count = len(b.materials)
        self.has_env = b.env_faces is not None


# ----------------------------------------------------------------------------------------------------------------------
# Camera + constants (BridgeCamera, Rtxpt/Shaders/PathTracer/PathTracerShared.h:109-141; Sample::UpdatePathTracerConstants,
# Rtxpt/Sample.cpp:1464-1556)
# ----------------------------------------------------------------------------------------------------------------------
def world_to_clip(cam):
    """SimpleViewConstants.matWorldToClip for a BridgeCamera block: row-major, row vector x matrix, D3D clip space (z in [0, 1])."""
    f = np.float32
    pos = np.array(cam.PosW[:], np.float32); W = np.array(cam.CameraW[:], np.float32); U = np.array(cam.CameraU[:], np.float32); V = np.array(cam.CameraV[:], np.float32)
    fwd = W / np.linalg.norm(W); right = U / np.linalg.norm(U); up = V / np.linalg.norm(V)
    tan_x, tan_y = float(np.linalg.norm(U) / np.linalg.norm(W)), float(np.linalg.norm(V) / np.linalg.norm(W))
    n, fa = float(cam.NearZ), float(cam.FarZ)
    view = np.eye(4, dtype=np.float64)
    view[:3, 0], view[:3, 1], view[:3, 2] = right, up, fwd
    view[3, :3] = [-np.dot(pos, right), -np.dot(pos, up), -np.dot(pos, fwd)]
    proj = np.zeros((4, 4), np.float64)
    proj[0, 0], proj[1, 1] = 1.0 / tan_x, 1.0 / tan_y
    proj[2, 2], proj[2, 3], proj[3, 2] = fa / (fa - n), 1.0, -n * fa / (fa - n)
    return (view @ proj).astype(f)


def make_realtime_constants(width, height, cam, prev_cam=None, active_planes=3, max_vertex_depth=14, bounce_count=None, allow_psr=True, sub_samples=1):
    """RtxptRealtimeConstants the way Sample::UpdatePathTracerConstants / UpdateViews fill them (Sample.cpp:1464-1480, :1529-1540): both views without
    the sub-pixel jitter offset, clipToWindowScale = (0.5 w, -0.5 h), maxStablePlaneVertexDepth = min(UI value, 15, bounceCount)."""
    rt = S.RealtimeConstants()
    rt.activeStablePlaneCount = active_planes
    rt.maxStablePlaneVertexDepth = min(max_vertex_depth, 15, bounce_count if bounce_count is not None else 15)
    rt.allowPrimarySurfaceReplacement = 1 if allow_psr else 0
    rt.subSampleCount = sub_samples
    rt.matWorldToClipNoOffset[:] = world_to_clip(cam).reshape(16).tolist()
    rt.prevMatWorldToClipNoOffset[:] = world_to_clip(prev_cam if prev_cam is not None else cam).reshape(16).tolist()
    rt.clipToWindowScale[:] = [0.5 * width, -0.5 * height]
    return rt


def world_to_view(cam):
    """SimpleViewConstants.matWorldToView for a BridgeCamera block (row-major, row vector x matrix; +z forward)."""
    pos = np.array(cam.PosW[:], np.float32); W = np.array(cam.CameraW[:], np.float32); U = np.array(cam.CameraU[:], np.float32); V = np.array(cam.CameraV[:], np.float32)
    fwd = W / np.linalg.norm(W); right = U / np.linalg.norm(U); up = V / np.linalg.norm(V)
    view = np.eye(4, dtype=np.float64)
    view[:3, 0], view[:3, 1], view[:3, 2] = right, up, fwd
    view[3, :3] = [-np.dot(pos, right), -np.dot(pos, up), -np.dot(pos, fwd)]
    return view.astype(np.float32)


def view_to_clip(cam):
    """SimpleViewConstants.matViewToClip of a BridgeCamera block (D3D, left-handed, z in [0, 1]); world_to_clip(cam) = world_to_view(cam) @ view_to_clip(cam)."""
    W = np.array(cam.CameraW[:], np.float32); U = np.array(cam.CameraU[:], np.float32); V = np.array(cam.CameraV[:], np.float32)
    tan_x, tan_y = float(np.linalg.norm(U) / np.linalg.norm(W)), float(np.linalg.norm(V) / np.linalg.norm(W))
    n, fa = float(cam.NearZ), float(cam.FarZ)
    proj = np.zeros((4, 4), np.float64)
    proj[0, 0], proj[1, 1] = 1.0 / tan_x, 1.0 / tan_y
    proj[2, 2], proj[2, 3], proj[3, 2] = fa / (fa - n), 1.0, -n * fa / (fa - n)
    return proj.astype(np.float32)


def make_denoiser_constants(cam, hit_distance_parameters=(3.0, 0.1, 20.0, -25.0), pre_exposed_gray_luminance=1.0, radiance_clamp_k=8.0, suppress_primary_indirect_specular_k=0.0):
    """RtxptDenoiserConstants: nrd::HitDistanceParameters defaults (NRDSettings.h:206-220), no tone mapping (preExposedGrayLuminance 1)."""
    k = S.DenoiserConstants()
    k.matWorldToView[:] = world_to_view(cam).reshape(16).tolist()
    k.hitDistanceParameters[:] = list(hit_distance_parameters)
    k.preExposedGrayLuminance = pre_exposed_gray_luminance; k.denoiserRadianceClampK = radiance_clamp_k
    k.stablePlanesSuppressPrimaryIndirectSpecularK = suppress_primary_indirect_specular_k
    return k


def make_reblur_frame(cam, prev_cam=None, frame_index=0, reset=False, ignore_motion_vectors=False, frame_time_ms=0.0):
    """RtxptReblurFrame from the current and the previous camera (un-jittered matrices, as NrdIntegration.cpp:375-408 passes them)."""
    f = S.ReblurFrame(); prev_cam = cam if prev_cam is None else prev_cam
    f.matWorldToView[:] = world_to_view(cam).reshape(16).tolist(); f.matViewToClip[:] = view_to_clip(cam).reshape(16).tolist()
    f.prevMatWorldToView[:] = world_to_view(prev_cam).reshape(16).tolist(); f.prevMatViewToClip[:] = view_to_clip(prev_cam).reshape(16).tolist()
    f.frameIndex = frame_index; f.resetHistory = 1 if reset else 0; f.ignoreMotionVectors = 1 if ignore_motion_vectors else 0; f.frameTimeMs = frame_time_ms
    return f


def generic_ts_address(x, y, plane, width, height):
    """GenericTSPixelToAddress (Utils.hlsli:337-352): 8x8 tiles, Morton order inside a tile; vectorised over numpy arrays."""
    x = np.asarray(x, np.uint32); y = np.asarray(y, np.uint32)
    line = ((width + 7) // 8) * 8; plane_stride = line * ((height + 7) // 8) * 8
    xi, yi = x % 8, y % 8
    def spread(v): v = (v | (v << 2)) & 0x33; return (v | (v << 1)) & 0x55
    morton = spread(xi) | (spread(yi) << 1)
    return ((x - xi) * 8 + (y - yi) * line + morton + plane * plane_stride).astype(np.uint32)


def bridge_camera(width, height, pos, direction, up, fov_y, near_z=0.1, far_z=1e7, focal_distance=10000.0, aperture_radius=0.0, jitter=(0.0, 0.0)):
    f = np.float32
    cam = S.CameraData()
    d = np.asarray(direction, np.float32); d = d / f(np.linalg.norm(d))
    W = (d * f(focal_distance)).astype(np.float32)
    U = np.cross(W, np.asarray(up, np.float32)).astype(np.float32); U = U / f(np.linalg.norm(U))
    V = np.cross(U, W).astype(np.float32); V = V / f(np.linalg.norm(V))
    aspect = f(width) / f(height)
    ulen = f(focal_distance) * f(math.tan(f(fov_y) * f(0.5))) * aspect
    vlen = f(focal_distance) * f(math.tan(f(fov_y) * f(0.5)))
    cam.PosW[:] = [float(x) for x in pos]; cam.NearZ = near_z; cam.FarZ = far_z
    cam.DirectionW[:] = d.tolist(); cam.CameraW[:] = W.tolist()
    cam.CameraU[:] = (U * ulen).astype(np.float32).tolist(); cam.CameraV[:] = (V * vlen).astype(np.float32).tolist()
    cam.FocalDistance, cam.AspectRatio, cam.ApertureRadius = focal_distance, float(aspect), aperture_radius
    cam.ViewportSize[:] = [width, height]
    cam.PixelConeSpreadAngle = float(f(math.atan(2.0 * math.tan(fov_y * 0.5) / height)))
    cam.Jitter[:] = [jitter[0], -jitter[1]]
    return cam


def make_constants(width, height, camera, bounce_count=6, diffuse_bounce_count=6, sample_base_index=0, nee=True, nee_type=2,
                   firefly_threshold=0.0, env_enabled=False, env_color=(1, 1, 1), russian_roulette=True, ld_sampler=True, nested_dielectrics=1,
                   aa_jitter=1.0, tex_lod_bias=-1.0, nee_candidates=5, nee_full=1, env_mip=2.0, distant_vs_local=1.0, approximate_mis=False):
    c = S.PathTracerConstants()
    c.imageWidth, c.imageHeight, c.sampleBaseIndex = width, height, sample_base_index
    c.perPixelJitterAAScale = aa_jitter
    c.bounceCount, c.diffuseBounceCount = bounce_count, diffuse_bounce_count
    c.EnvironmentMapDiffuseSampleMIPLevel, c.texLODBias = env_mip, tex_lod_bias
    c.fireflyFilterThreshold = firefly_threshold
    c.NEEEnabled, c.NEEType, c.NEECandidateSamples, c.NEEFullSamples = int(nee), nee_type, nee_candidates, nee_full
    c.enableRussianRoulette, c.enableLDSamplerForBSDF, c.nestedDielectricsQuality = int(russian_roulette), int(ld_sampler), nested_dielectrics
    c.camera = camera
    ident = [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0]
    c.envMap.Transform[:] = ident; c.envMap.InvTransform[:] = ident
    c.envMap.ColorMultiplier[:] = env_color; c.envMap.Enabled = 1.0 if env_enabled else 0.0
    c.distantVsLocalImportance = distant_vs_local
    c.useApproximateMIS = int(approximate_mis)
    return c
