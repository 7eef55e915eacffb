"""ctypes bindings of ReBLUR with panel settings - TEST INFRASTRUCTURE ONLY: the oracle's instance that carries settings (oracle/reblur_settings.mk:
liboracle_reblur_settings.so, oracle/reblur_settings.h) and the host build of the product's passes under settings (tests/emu/reblur_settings.mk: libreblur_settings_emu.so).
Same call shapes as oracle_lib.Reblur.denoise and host_build_lib.ReblurPort.denoise, plus set(settings) with a structs.ReblurSettings."""
import ctypes as C
import os
import subprocess
import numpy as np
from rtxpt_b200 import structs as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_PATH = os.path.join(ROOT, "oracle", "_build", "reblur_settings", "liboracle_reblur_settings.so")
EMU_PATH = os.path.join(ROOT, "tests", "emu", "_build", "libreblur_settings_emu.so")
_libs = {}


def build():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "-f", "reblur_settings.mk"], check=True)
    subprocess.run(["make", "-C", os.path.join(ROOT, "tests", "emu"), "-s", "-f", "reblur_settings.mk"], check=True)


def _lib(which):
    if which not in _libs:
        build()
        if which == "oracle":
            L = C.CDLL(ORACLE_PATH)
            L.oracle_reblur_settings_create.restype = C.c_void_p; L.oracle_reblur_settings_destroy.argtypes = [C.c_void_p]
            L.oracle_reblur_settings_set.argtypes = [C.c_void_p, C.POINTER(S.ReblurSettings)]; L.oracle_reblur_settings_set.restype = C.c_int
            L.oracle_reblur_settings_denoise.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 4 + [C.c_uint32, C.c_int] + [C.c_void_p] * 9
            L.oracle_reblur_settings_denoise.restype = C.c_int
        else:
            L = C.CDLL(EMU_PATH)
            L.rbs_emu_create.restype = C.c_void_p; L.rbs_emu_destroy.argtypes = [C.c_void_p]
            L.rbs_emu_set_settings.argtypes = [C.c_void_p, C.POINTER(S.ReblurSettings)]; L.rbs_emu_set_settings.restype = C.c_int
            L.rbs_emu_denoise.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(S.ReblurFrame)] + [C.c_void_p] * 9; L.rbs_emu_denoise.restype = C.c_int
        _libs[which] = L
    return _libs[which]


def _arrays(view_z, normal_roughness, diff, spec, motion, disocclusion_mix):
    c = lambda a, t: None if a is None else np.ascontiguousarray(a, t)
    return c(view_z, np.float32), c(normal_roughness, np.uint32), c(diff, np.float16), c(spec, np.float16), c(motion, np.float16), c(disocclusion_mix, np.uint8)


def _ptr(a): return None if a is None else a.ctypes.data


class OracleReblur:
    """One oracle ReBLUR instance with settings (RTXPT's until set); history persists between denoise calls."""
    def __init__(self): self.h = _lib("oracle").oracle_reblur_settings_create()

    def close(self):
        if self.h: _lib("oracle").oracle_reblur_settings_destroy(self.h); self.h = None

    def __del__(self): self.close()

    def set(self, settings): assert _lib("oracle").oracle_reblur_settings_set(self.h, C.byref(settings)) == 0

    def denoise(self, world_to_view, view_to_clip, frame_index, view_z, normal_roughness, diff, spec, prev_world_to_view=None, prev_view_to_clip=None, motion=None, disocclusion_mix=None, reset=False):
        H, W = view_z.shape
        m0, m1 = np.ascontiguousarray(world_to_view, np.float32), np.ascontiguousarray(view_to_clip, np.float32)
        p0 = m0 if prev_world_to_view is None else np.ascontiguousarray(prev_world_to_view, np.float32); p1 = m1 if prev_view_to_clip is None else np.ascontiguousarray(prev_view_to_clip, np.float32)
        vz, nr, d, s, mv, mix = _arrays(view_z, normal_roughness, diff, spec, motion, disocclusion_mix)
        od = np.zeros((H, W, 4), np.float16); os_ = np.zeros((H, W, 4), np.float16); frames = np.zeros((H, W, 2), np.float32)
        rc = _lib("oracle").oracle_reblur_settings_denoise(self.h, W, H, _ptr(m0), _ptr(m1), _ptr(p0), _ptr(p1), frame_index, int(reset), _ptr(vz), _ptr(nr), _ptr(mv), _ptr(mix), _ptr(d), _ptr(s),
                                                           _ptr(od), _ptr(os_), _ptr(frames))
        assert rc == 0
        return od, os_, frames


class PortReblur:
    """One instance of the host-compiled product passes with settings (RTXPT's until set); set() returns what rtxpt_b200_set_reblur_settings would: 0 or -1, settings kept."""
    def __init__(self): self.h = _lib("emu").rbs_emu_create()

    def close(self):
        if self.h: _lib("emu").rbs_emu_destroy(self.h); self.h = None

    def __del__(self): self.close()

    def set(self, settings): return _lib("emu").rbs_emu_set_settings(self.h, C.byref(settings))

    def denoise(self, frame, view_z, normal_roughness, diff, spec, motion=None, disocclusion_mix=None):
        H, W = view_z.shape
        vz, nr, d, s, mv, mix = _arrays(view_z, normal_roughness, diff, spec, motion, disocclusion_mix)
        od = np.zeros((H, W, 4), np.float16); os_ = np.zeros((H, W, 4), np.float16); frames = np.zeros((H, W, 2), np.float32)
        rc = _lib("emu").rbs_emu_denoise(self.h, W, H, C.byref(frame), _ptr(vz), _ptr(nr), _ptr(mv), _ptr(mix), _ptr(d), _ptr(s), _ptr(od), _ptr(os_), _ptr(frames))
        assert rc == 0
        return od, os_, frames
